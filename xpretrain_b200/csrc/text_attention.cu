// CLIP text-tower self-attention, forward and backward: CLIPAttention.forward, CLIP_ViP.py:266-330, with the
// additive causal mask (-inf above the diagonal, :788-797) and the additive padding mask (finfo.min on masked
// keys, :50-61,760).  Sequences are <= 77 tokens and the whole tower is 0.6 % of the FLOPs, so this is a
// latency-oriented CUDA-core kernel: one CTA per (batch, head), fp32 math, probabilities saved for backward.
#include <float.h>

#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

constexpr int TA_HD = 64;
constexpr int TA_MAXL = 96;
constexpr int TA_LDS = TA_HD + 1;  // padded fp32 row

__device__ __forceinline__ void ta_load_rows(const __nv_bfloat16* __restrict__ src, long long ld, int Lt, float* dst) {
  // src: Lt rows of 64 bf16 (row stride ld) -> dst [Lt][65] fp32
  for (int idx = threadIdx.x; idx < Lt * 8; idx += blockDim.x) {
    const int r = idx >> 3, ch = idx & 7;
    const uint4 u = *reinterpret_cast<const uint4*>(src + static_cast<long long>(r) * ld + ch * 8);
    float* o = dst + r * TA_LDS + ch * 8;
    o[0] = bf16_lo(u.x); o[1] = bf16_hi(u.x); o[2] = bf16_lo(u.y); o[3] = bf16_hi(u.y);
    o[4] = bf16_lo(u.z); o[5] = bf16_hi(u.z); o[6] = bf16_lo(u.w); o[7] = bf16_hi(u.w);
  }
}

// grid (H, B), 128 threads.  qkv bf16 [B*Lt, 3C]; mask int64 [B, Lt] (1 = keep); out bf16 [B*Lt, C];
// probs f32 [B, H, Lt, Lt].
__global__ void __launch_bounds__(128)
text_attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, const long long* __restrict__ mask,
                     __nv_bfloat16* __restrict__ out, float* __restrict__ probs, int Lt, int C, int H) {
  extern __shared__ float sm[];
  float* sq = sm;
  float* sk = sq + Lt * TA_LDS;
  float* sv = sk + Lt * TA_LDS;
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ld = 3LL * C;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * Lt * ld + h * TA_HD;
  ta_load_rows(base, ld, Lt, sq);
  ta_load_rows(base + C, ld, Lt, sk);
  ta_load_rows(base + 2 * C, ld, Lt, sv);
  __syncthreads();
  float* pr = probs + (static_cast<long long>(b) * H + h) * Lt * Lt;
  for (int i = warp; i < Lt; i += 4) {
    float s[3];
    float mx = -INFINITY;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int j = lane + u * 32;
      s[u] = -INFINITY;
      if (j < Lt) {
        float acc = 0.f;
#pragma unroll 16
        for (int dd = 0; dd < TA_HD; ++dd) acc = fmaf(sq[i * TA_LDS + dd], sk[j * TA_LDS + dd], acc);
        // reference order: scores + causal mask, then + padding mask (fp32 adds, CLIP_ViP.py:288-300)
        if (j > i) acc += -INFINITY;
        if (mask != nullptr && mask[static_cast<long long>(b) * Lt + j] == 0) acc += -FLT_MAX;
        s[u] = acc;
      }
      mx = fmaxf(mx, s[u]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      s[u] = (lane + u * 32 < Lt) ? __expf(s[u] - mx) : 0.f;
      sum += s[u];
    }
    sum = warp_sum(sum);
    const float inv = 1.f / sum;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      s[u] *= inv;
      if (lane + u * 32 < Lt) pr[static_cast<long long>(i) * Lt + lane + u * 32] = s[u];
    }
    float o0 = 0.f, o1 = 0.f;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      for (int jj = 0; jj < 32; ++jj) {
        const int j = u * 32 + jj;
        if (j >= Lt) break;
        const float p = __shfl_sync(0xffffffffu, s[u], jj);
        o0 = fmaf(p, sv[j * TA_LDS + lane], o0);
        o1 = fmaf(p, sv[j * TA_LDS + lane + 32], o1);
      }
    }
    __nv_bfloat16* orow = out + (static_cast<long long>(b) * Lt + i) * C + h * TA_HD;
    orow[lane] = __float2bfloat16(o0);
    orow[lane + 32] = __float2bfloat16(o1);
  }
}

// grid (H, B), 128 threads.  dqkv bf16 [B*Lt, 3C]; the dq third carries q_scale (CLIP_ViP.py:269).
__global__ void __launch_bounds__(128)
text_attn_bwd_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout,
                     const float* __restrict__ probs, __nv_bfloat16* __restrict__ dqkv, int Lt, int C, int H,
                     float q_scale) {
  extern __shared__ float sm[];
  float* sq = sm;
  float* sk = sq + Lt * TA_LDS;
  float* sv = sk + Lt * TA_LDS;
  float* sdo = sv + Lt * TA_LDS;
  float* sp = sdo + Lt * TA_LDS;       // [Lt][Lt+1] probabilities
  float* sds = sp + Lt * (Lt + 1);     // [Lt][Lt+1] dS
  const int h = blockIdx.x, b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ld = 3LL * C;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * Lt * ld + h * TA_HD;
  ta_load_rows(base, ld, Lt, sq);
  ta_load_rows(base + C, ld, Lt, sk);
  ta_load_rows(base + 2 * C, ld, Lt, sv);
  ta_load_rows(dout + static_cast<long long>(b) * Lt * C + h * TA_HD, C, Lt, sdo);
  const float* pr = probs + (static_cast<long long>(b) * H + h) * Lt * Lt;
  for (int idx = threadIdx.x; idx < Lt * Lt; idx += blockDim.x) sp[(idx / Lt) * (Lt + 1) + idx % Lt] = pr[idx];
  __syncthreads();
  // dP = dO V^T ; dS = P * (dP - rowsum(P * dP))
  for (int i = warp; i < Lt; i += 4) {
    float dp[3], dot = 0.f;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int j = lane + u * 32;
      dp[u] = 0.f;
      if (j < Lt) {
        float acc = 0.f;
#pragma unroll 16
        for (int dd = 0; dd < TA_HD; ++dd) acc = fmaf(sdo[i * TA_LDS + dd], sv[j * TA_LDS + dd], acc);
        dp[u] = acc;
        dot += acc * sp[i * (Lt + 1) + j];
      }
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int j = lane + u * 32;
      if (j < Lt) sds[i * (Lt + 1) + j] = sp[i * (Lt + 1) + j] * (dp[u] - dot);
    }
  }
  __syncthreads();
  for (int r = warp; r < Lt; r += 4) {
    // dQ[r] = sum_j dS[r][j] K[j];  dK[r] = sum_i dS[i][r] Q[i];  dV[r] = sum_i P[i][r] dO[i]
    float dq0 = 0.f, dq1 = 0.f, dk0 = 0.f, dk1 = 0.f, dv0 = 0.f, dv1 = 0.f;
    for (int j = 0; j < Lt; ++j) {
      const float a = sds[r * (Lt + 1) + j];
      dq0 = fmaf(a, sk[j * TA_LDS + lane], dq0);
      dq1 = fmaf(a, sk[j * TA_LDS + lane + 32], dq1);
      const float bt = sds[j * (Lt + 1) + r];
      dk0 = fmaf(bt, sq[j * TA_LDS + lane], dk0);
      dk1 = fmaf(bt, sq[j * TA_LDS + lane + 32], dk1);
      const float pt = sp[j * (Lt + 1) + r];
      dv0 = fmaf(pt, sdo[j * TA_LDS + lane], dv0);
      dv1 = fmaf(pt, sdo[j * TA_LDS + lane + 32], dv1);
    }
    __nv_bfloat16* row = dqkv + (static_cast<long long>(b) * Lt + r) * ld + h * TA_HD;
    row[lane] = __float2bfloat16(dq0 * q_scale);
    row[lane + 32] = __float2bfloat16(dq1 * q_scale);
    row[C + lane] = __float2bfloat16(dk0);
    row[C + lane + 32] = __float2bfloat16(dk1);
    row[2 * C + lane] = __float2bfloat16(dv0);
    row[2 * C + lane + 32] = __float2bfloat16(dv1);
  }
}

}  // namespace xp

using namespace xp;

extern "C" int xp_text_attention_fwd(const void* qkv, const int64_t* mask, void* out, float* probs, int32_t B, int32_t H,
                                     int32_t Lt, int32_t C, void* stream) {
  XP_ENTER(qkv);
  if (C != H * TA_HD) return fail("xp_text_attention_fwd: head_dim must be 64");
  if (Lt > TA_MAXL || Lt < 1) return fail("xp_text_attention_fwd: 1 <= Lt <= 96");
  const int smem = 3 * Lt * TA_LDS * 4;
  if (smem_limit<text_attn_fwd_kernel>(3 * TA_MAXL * TA_LDS * 4)) return -1;
  text_attn_fwd_kernel<<<dim3(H, B), 128, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(qkv), reinterpret_cast<const long long*>(mask), static_cast<__nv_bfloat16*>(out),
      probs, Lt, C, H);
  XP_CHECK_LAUNCH("text_attn_fwd_kernel");
  return 0;
}

extern "C" int xp_text_attention_bwd(const void* qkv, const void* dout, const float* probs, void* dqkv, int32_t B,
                                     int32_t H, int32_t Lt, int32_t C, float q_scale, void* stream) {
  XP_ENTER(qkv);
  if (C != H * TA_HD) return fail("xp_text_attention_bwd: head_dim must be 64");
  if (Lt > TA_MAXL || Lt < 1) return fail("xp_text_attention_bwd: 1 <= Lt <= 96");
  const int smem = (4 * Lt * TA_LDS + 2 * Lt * (Lt + 1)) * 4;
  if (smem_limit<text_attn_bwd_kernel>((4 * TA_MAXL * TA_LDS + 2 * TA_MAXL * (TA_MAXL + 1)) * 4)) return -1;
  text_attn_bwd_kernel<<<dim3(H, B), 128, smem, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(qkv), static_cast<const __nv_bfloat16*>(dout), probs,
      static_cast<__nv_bfloat16*>(dqkv), Lt, C, H, q_scale);
  XP_CHECK_LAUNCH("text_attn_bwd_kernel");
  return 0;
}
