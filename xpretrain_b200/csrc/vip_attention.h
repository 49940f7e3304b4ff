// Shapes shared by the two proxy-token (ViP) attention translation units: vip_attention.cu (frames of M + L <= 208 rows,
// staged whole) and vip_attention_long.cu (longer frames, streamed in 64-row blocks).  Both write the same per-frame
// partials of the M global rows, which vip_attention.cu's combine kernels merge.
#pragma once
#include <cuda_runtime.h>

namespace xp {

constexpr int VIP_STAGED_MAX_ROWS = 208;   // M + L up to this runs the staged kernel, longer frames the streamed one

struct AttnDims {
  int B, H, T, L, M;
  long long S;       // M + T*L
  long long ld_qkv;  // 3*C
  long long ld_o;    // C
  int C;
};

__device__ __forceinline__ long long token_row(const AttnDims& d, int b, int t, int i) {
  return static_cast<long long>(b) * d.S + (i < d.M ? i : d.M + static_cast<long long>(t) * d.L + (i - d.M));
}

// Streamed kernels for M + L > VIP_STAGED_MAX_ROWS.  Forward: the frame rows of out and lse, and the per-frame partials
// part [B, H, T, M, 66] of the global queries.  Backward: the frame rows of dqkv and the per-frame partials
// gpart [B, H, T, M, 3, 64] of the global rows' dq / dk / dv.  The caller launches the combine kernels.
int vip_long_attn_fwd(const AttnDims& d, const void* qkv, void* out, float* lse, float* part, cudaStream_t st);
int vip_long_attn_bwd(const AttnDims& d, const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                      float* gpart, float q_scale, cudaStream_t st);

}  // namespace xp
