// Token assembly of HD-VILA's TimeSformer (BASELINE.json config #4) and its backward.
//
// Reference: TimeSformer.forward timesformer.py:481-509 — the [B,T,C,H,W] feature maps are flattened to
// '(b t) (h w) c', the (interpolated) positional table is added, then '(b n) t m' + the (interpolated) time table,
// then 'b (n t) m'.  Net effect: token (b, p = h*W + w, t) = x[b, t, :, p] + pos[p, :] + time[t, :], rows ordered
// (h w t).  That is a [C, HW] -> [HW, C] transpose per (b, t) with two table adds; three rearrange copies and two
// broadcast adds in the reference, one pass here (32x32 shared-memory tiles, coalesced on both sides).
// Backward: d x[b,t,c,p] = d token[(b,p,t), c] — the transposed copy; the table gradients are column sums of the token
// gradient (xp_colsum_bf16 on reshaped views, see modeling/timesformer.py).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

// grid (ceil(HW/32), ceil(C/32), B*T), block (32, 8)
template <typename T>
__global__ void __launch_bounds__(256)
tsf_embed_fwd_kernel(const T* __restrict__ x, const float* __restrict__ pos, const float* __restrict__ time,
                     __nv_bfloat16* __restrict__ tok, int Tn, int C, int HW) {
  __shared__ float tile[32][33];
  const int bt = blockIdx.z, b = bt / Tn, t = bt - b * Tn;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const T* src = x + static_cast<long long>(bt) * C * HW;
#pragma unroll
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, p = p0 + threadIdx.x;
    tile[j][threadIdx.x] = (c < C && p < HW) ? to_f32<T>(src[static_cast<long long>(c) * HW + p]) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    if (p < HW && c < C) {
      float v = tile[threadIdx.x][j];   // null tables: plain tokenisation (used for the output gradient)
      if (pos != nullptr) v += pos[static_cast<long long>(p) * C + c];
      if (time != nullptr) v += time[static_cast<long long>(t) * C + c];
      tok[((static_cast<long long>(b) * HW + p) * Tn + t) * C + c] = __float2bfloat16(v);
    }
  }
}

// dx[b,t,c,p] = d_tok[(b,p,t), c];  grid (ceil(HW/32), ceil(C/32), B*T), block (32, 8)
template <typename T>
__global__ void __launch_bounds__(256)
tsf_embed_bwd_kernel(const __nv_bfloat16* __restrict__ d_tok, T* __restrict__ dx, int Tn, int C, int HW) {
  __shared__ float tile[32][33];
  const int bt = blockIdx.z, b = bt / Tn, t = bt - b * Tn;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
#pragma unroll
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int p = p0 + j, c = c0 + threadIdx.x;
    tile[j][threadIdx.x] =
        (p < HW && c < C) ? __bfloat162float(d_tok[((static_cast<long long>(b) * HW + p) * Tn + t) * C + c]) : 0.f;
  }
  __syncthreads();
  T* dst = dx + static_cast<long long>(bt) * C * HW;
#pragma unroll
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int c = c0 + j, p = p0 + threadIdx.x;
    if (c < C && p < HW) dst[static_cast<long long>(c) * HW + p] = from_f32<T>(tile[threadIdx.x][j]);
  }
}

// out[b,t,c,p] = tok[(b,p,t), c]: the reference returns x.reshape(B,H,W,T,C).permute(0,3,4,1,2) (timesformer.py:523) as a
// strided view; callers that need it contiguous (or in fp32) get it from the same transposed copy as the backward.

}  // namespace xp

using namespace xp;

extern "C" int xp_tsf_embed_fwd(const void* x, int32_t x_dtype, const float* pos, const float* time, void* tokens,
                                int32_t B, int32_t T, int32_t C, int32_t HW, void* stream) {
  XP_ENTER(x);
  if (B <= 0 || T <= 0 || C <= 0 || HW <= 0) return fail("xp_tsf_embed_fwd: empty shape");
  if (static_cast<long long>(B) * T > 65535) return fail("xp_tsf_embed_fwd: B*T > 65535");
  const dim3 grid((HW + 31) / 32, (C + 31) / 32, B * T), block(32, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* tok = static_cast<__nv_bfloat16*>(tokens);
  return dispatch_dtype(x_dtype, "xp_tsf_embed_fwd: x_dtype must be XP_DTYPE_F32 / BF16 / F16", [&](auto t) {
    using E = decltype(t);
    tsf_embed_fwd_kernel<E><<<grid, block, 0, st>>>(static_cast<const E*>(x), pos, time, tok, T, C, HW);
    XP_CHECK_LAUNCH("tsf_embed_fwd_kernel");
    return 0;
  });
}

extern "C" int xp_tsf_untokenize(const void* tokens, void* x, int32_t x_dtype, int32_t B, int32_t T, int32_t C, int32_t HW,
                                 void* stream) {
  XP_ENTER(tokens);
  if (B <= 0 || T <= 0 || C <= 0 || HW <= 0) return fail("xp_tsf_untokenize: empty shape");
  if (static_cast<long long>(B) * T > 65535) return fail("xp_tsf_untokenize: B*T > 65535");
  const dim3 grid((HW + 31) / 32, (C + 31) / 32, B * T), block(32, 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* tok = static_cast<const __nv_bfloat16*>(tokens);
  return dispatch_dtype(x_dtype, "xp_tsf_untokenize: x_dtype must be XP_DTYPE_F32 / BF16 / F16", [&](auto t) {
    using E = decltype(t);
    tsf_embed_bwd_kernel<E><<<grid, block, 0, st>>>(tok, static_cast<E*>(x), T, C, HW);
    XP_CHECK_LAUNCH("tsf_embed_bwd_kernel");
    return 0;
  });
}
