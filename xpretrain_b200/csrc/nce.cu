// In-batch video<->text InfoNCE with a learnable temperature: NCELearnableTempLoss.forward, loss.py:134-141,
// on the rank-major gathered embeddings (hvd.allgather, run_pretrain.py:344-345).
//
//   Z = exp(logit_scale) * V T^T                     [N, N]   (rows = videos)
//   loss = mean_i(LSE_j Z_ij - Z_ii) + mean_j(LSE_i Z_ij - Z_jj)        (SUM of the two CEs, no 1/2)
//   G = dL/dZ = (softmax_rows(Z) + softmax_cols(Z) - 2I) / N
//   dV = s G T,  dT = s G^T V,  d logit_scale = sum_ij G_ij Z_ij         (SURVEY.md §8e closed form)
//
// The two GEMM-shaped steps run on the wgmma GEMM (gemm.cu).  To keep fp32-level logits out of bf16
// tensor-core inputs, V and T are split into bf16 hi + lo parts and the three significant cross terms are
// concatenated along K:  [Vh | Vh | Vl] . [Th | Tl | Th]^T  (K = 3d), i.e. one GEMM, ~2^-16 relative error.
// The kernels here are the prep / softmax / gradient pieces around those GEMMs.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

// a3[r] = [hi | hi | lo], b3[r] = [hi | lo | hi] selected by `pattern` (0 -> A layout, 1 -> B layout); hi_out = hi
__global__ void __launch_bounds__(128)
nce_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ x3, __nv_bfloat16* __restrict__ hi_out,
                 int d, int pattern) {
  const long long r = blockIdx.x;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const float v = x[r * d + c];
    const __nv_bfloat16 hi = __float2bfloat16(v);
    const __nv_bfloat16 lo = __float2bfloat16(v - __bfloat162float(hi));
    __nv_bfloat16* o = x3 + r * 3 * d;
    o[c] = hi;
    o[d + c] = pattern == 0 ? hi : lo;
    o[2 * d + c] = pattern == 0 ? lo : hi;
    if (hi_out) hi_out[r * d + c] = hi;
  }
}

// lse[i] = log sum_j exp(s * Z[i*si + j*sj]) ; one warp per output, 4 per CTA.
__global__ void __launch_bounds__(128)
nce_lse_kernel(const float* __restrict__ z, const float* __restrict__ logit_scale, float* __restrict__ lse, int N,
               long long si, long long sj) {
  const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= N) return;
  const float s = expf(*logit_scale);
  float mx = -INFINITY;
  for (int j = lane; j < N; j += 32) mx = fmaxf(mx, s * z[i * si + j * sj]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int j = lane; j < N; j += 32) sum += expf(s * z[i * si + j * sj] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) lse[i] = mx + logf(sum);
}

// One CTA per row i: G'[i,j] = s * G[i,j] (bf16), loss += (lse_r[i] + lse_c[i] - 2 Z_ii)/N, dscale += sum_j G_ij Z_ij.
__global__ void __launch_bounds__(128)
nce_grad_kernel(const float* __restrict__ z, const float* __restrict__ logit_scale, const float* __restrict__ lse_r,
                const float* __restrict__ lse_c, __nv_bfloat16* __restrict__ g_scaled, float* __restrict__ loss,
                float* __restrict__ dscale, int N, long long ld) {
  __shared__ float red[4];
  const int i = blockIdx.x;
  const float s = expf(*logit_scale);
  const float inv_n = 1.f / N;
  float acc = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float zz = s * z[static_cast<long long>(i) * ld + j];
    float g = (expf(zz - lse_r[i]) + expf(zz - lse_c[j]) - (i == j ? 2.f : 0.f)) * inv_n;
    acc += g * zz;
    if (g_scaled) g_scaled[static_cast<long long>(i) * ld + j] = __float2bfloat16(g * s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (dscale) atomicAdd(dscale, red[0] + red[1] + red[2] + red[3]);
    const float zii = s * z[static_cast<long long>(i) * ld + i];
    atomicAdd(loss, (lse_r[i] + lse_c[i] - 2.f * zii) * inv_n);
  }
}

// ---------------------------------------------------------------------------------------------------------
// NCELearnableTempLoss_vsc_fc, loss.py:288-324 (six cross-entropies over A = s V T^T, B = s V C^T, D = s I C^T):
//   columns of A, columns of B, columns of D, rows of D, and per row i the two mixed softmaxes
//     r3_i = LSE(A_i,: U B_i,j!=i)  with target A_ii        r4_i = LSE(A_i,j!=i U B_i,:)  with target B_ii.
// Row statistics r3, r4, rD: one warp per row.
__global__ void __launch_bounds__(128)
nce3_rowstats_kernel(const float* __restrict__ za, const float* __restrict__ zb, const float* __restrict__ zd,
                     const float* __restrict__ logit_scale, float* __restrict__ r3, float* __restrict__ r4,
                     float* __restrict__ rd, int N, long long ld) {
  const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= N) return;
  const float s = expf(*logit_scale);
  const float* a = za + static_cast<long long>(i) * ld;
  const float* b = zb + static_cast<long long>(i) * ld;
  const float* d = zd + static_cast<long long>(i) * ld;
  float mab = -INFINITY, md = -INFINITY;
  for (int j = lane; j < N; j += 32) {
    mab = fmaxf(mab, fmaxf(s * a[j], s * b[j]));
    md = fmaxf(md, s * d[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mab = fmaxf(mab, __shfl_xor_sync(0xffffffffu, mab, o));
    md = fmaxf(md, __shfl_xor_sync(0xffffffffu, md, o));
  }
  float s3 = 0.f, s4 = 0.f, sd = 0.f;
  for (int j = lane; j < N; j += 32) {
    const float ea = expf(s * a[j] - mab), eb = expf(s * b[j] - mab);
    s3 += ea + (j == i ? 0.f : eb);
    s4 += (j == i ? 0.f : ea) + eb;
    sd += expf(s * d[j] - md);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s3 += __shfl_xor_sync(0xffffffffu, s3, o);
    s4 += __shfl_xor_sync(0xffffffffu, s4, o);
    sd += __shfl_xor_sync(0xffffffffu, sd, o);
  }
  if (lane == 0) {
    r3[i] = mab + logf(s3);
    r4[i] = mab + logf(s4);
    rd[i] = md + logf(sd);
  }
}

// One CTA per row i: the three gradient matrices (times s, bf16), the loss and d logit_scale = sum G . Z.
__global__ void __launch_bounds__(128)
nce3_grad_kernel(const float* __restrict__ za, const float* __restrict__ zb, const float* __restrict__ zd,
                 const float* __restrict__ logit_scale, const float* __restrict__ ca, const float* __restrict__ cb,
                 const float* __restrict__ cd, const float* __restrict__ r3, const float* __restrict__ r4,
                 const float* __restrict__ rd, __nv_bfloat16* __restrict__ ga, __nv_bfloat16* __restrict__ gb,
                 __nv_bfloat16* __restrict__ gd, float* __restrict__ loss, float* __restrict__ dscale, int N, long long ld) {
  __shared__ float red[4];
  const int i = blockIdx.x;
  const float s = expf(*logit_scale);
  const float inv_n = 1.f / N;
  const float r3i = r3[i], r4i = r4[i], rdi = rd[i];
  const long long row = static_cast<long long>(i) * ld;
  float acc = 0.f;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float a = s * za[row + j], b = s * zb[row + j], d = s * zd[row + j];
    const bool diag = (i == j);
    const float g_a = (expf(a - ca[j]) + expf(a - r3i) + (diag ? 0.f : expf(a - r4i)) - (diag ? 2.f : 0.f)) * inv_n;
    const float g_b = (expf(b - cb[j]) + (diag ? 0.f : expf(b - r3i)) + expf(b - r4i) - (diag ? 2.f : 0.f)) * inv_n;
    const float g_d = (expf(d - cd[j]) + expf(d - rdi) - (diag ? 2.f : 0.f)) * inv_n;
    acc += g_a * a + g_b * b + g_d * d;
    ga[row + j] = __float2bfloat16(g_a * s);
    gb[row + j] = __float2bfloat16(g_b * s);
    gd[row + j] = __float2bfloat16(g_d * s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (dscale) atomicAdd(dscale, red[0] + red[1] + red[2] + red[3]);
    const float aii = s * za[row + i], bii = s * zb[row + i], dii = s * zd[row + i];
    atomicAdd(loss, (ca[i] + r3i - 2.f * aii + cb[i] + r4i - 2.f * bii + cd[i] + rdi - 2.f * dii) * inv_n);
  }
}

}  // namespace xp

using namespace xp;

extern "C" int xp_nce_vsc_fc(const float* za, const float* zb, const float* zd, const float* logit_scale, float* stats,
                             void* ga_bf16, void* gb_bf16, void* gd_bf16, float* loss, float* d_logit_scale, int32_t N,
                             int64_t ld, void* stream) {
  XP_ENTER(za);
  if (N <= 0) return fail("xp_nce_vsc_fc: N must be positive");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float *ca = stats, *cb = stats + N, *cd = stats + 2 * N, *r3 = stats + 3 * N, *r4 = stats + 4 * N, *rd = stats + 5 * N;
  XP_CHECK_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
  const int g4 = (N + 3) / 4;
  nce_lse_kernel<<<g4, 128, 0, st>>>(za, logit_scale, ca, N, 1, ld);
  XP_CHECK_LAUNCH("nce_lse_kernel");
  nce_lse_kernel<<<g4, 128, 0, st>>>(zb, logit_scale, cb, N, 1, ld);
  XP_CHECK_LAUNCH("nce_lse_kernel");
  nce_lse_kernel<<<g4, 128, 0, st>>>(zd, logit_scale, cd, N, 1, ld);
  XP_CHECK_LAUNCH("nce_lse_kernel");
  nce3_rowstats_kernel<<<g4, 128, 0, st>>>(za, zb, zd, logit_scale, r3, r4, rd, N, ld);
  XP_CHECK_LAUNCH("nce3_rowstats_kernel");
  nce3_grad_kernel<<<N, 128, 0, st>>>(za, zb, zd, logit_scale, ca, cb, cd, r3, r4, rd,
                                      static_cast<__nv_bfloat16*>(ga_bf16), static_cast<__nv_bfloat16*>(gb_bf16),
                                      static_cast<__nv_bfloat16*>(gd_bf16), loss, d_logit_scale, N, ld);
  XP_CHECK_LAUNCH("nce3_grad_kernel");
  return 0;
}

extern "C" int xp_nce_split(const float* x, void* x3_bf16, void* hi_bf16, int32_t rows, int32_t d, int32_t pattern,
                            void* stream) {
  XP_ENTER(x);
  if (rows <= 0) return 0;
  nce_split_kernel<<<rows, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<__nv_bfloat16*>(x3_bf16), static_cast<__nv_bfloat16*>(hi_bf16), d, pattern);
  XP_CHECK_LAUNCH("nce_split_kernel");
  return 0;
}

extern "C" int xp_nce_softmax_grad(const float* z, const float* logit_scale, float* lse_rows, float* lse_cols,
                                   void* g_scaled_bf16, float* loss, float* d_logit_scale, int32_t N, int64_t ld,
                                   void* stream) {
  XP_ENTER(z);
  if (N <= 0) return fail("xp_nce_softmax_grad: N must be positive");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  XP_CHECK_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
  nce_lse_kernel<<<(N + 3) / 4, 128, 0, st>>>(z, logit_scale, lse_rows, N, ld, 1);
  XP_CHECK_LAUNCH("nce_lse_kernel");
  nce_lse_kernel<<<(N + 3) / 4, 128, 0, st>>>(z, logit_scale, lse_cols, N, 1, ld);
  XP_CHECK_LAUNCH("nce_lse_kernel");
  nce_grad_kernel<<<N, 128, 0, st>>>(z, logit_scale, lse_rows, lse_cols, static_cast<__nv_bfloat16*>(g_scaled_bf16),
                                     loss, d_logit_scale, N, ld);
  XP_CHECK_LAUNCH("nce_grad_kernel");
  return 0;
}
