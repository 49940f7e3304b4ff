// Retrieval evaluation on the device (SURVEY.md §8f.3).
//
// Reference: validate() CLIP-ViP/src/pretrain/run_pretrain.py:128-200 and tasks/run_video_retrieval.py:150-172 move every
// feature batch to the host and run numpy there: cal_cossim (utils/metrics.py:3-5), the DSL re-weighting
// sim * softmax(100 * sim, axis=0) (run_video_retrieval.py:169-170, np_softmax metrics.py:7-39) and compute_metrics
// (metrics.py:41-53: a full sort of every row to find the rank of the diagonal).  Here the O(N^2 d) and O(N^2) parts
// stay on the GPU and only two int32 vectors per direction travel to the host:
//   sim_f32_kernel      sim = A B^T in fp32 FFMA (fp32 like numpy's dot — ranks must not depend on a bf16 rounding)
//   dsl_*               column-wise softmax re-weighting, in place
//   rank_counts_kernel  for row (or column) i: how many entries are strictly larger than / equal to the diagonal entry;
//                       the rank list of compute_metrics (including its tie quirk) follows from those two counts.  The
//                       reference finds the diagonal's positions as zeros of sort(-x) - diag(-x), which is never 0 when
//                       the diagonal is NaN or +-inf (NaN, or inf - inf): such a query has no equal entries.
// Integer outputs are exact functions of the similarity matrix they are computed from.
#include "../../include/xpretrain_b200.h"
#include "common.h"

namespace xp {

constexpr int SIM_T = 64;   // output tile
constexpr int SIM_K = 16;

// grid (ceil(Nb/64), ceil(Na/64)), 256 threads, each thread a 4x4 block of the 64x64 tile
__global__ void __launch_bounds__(256)
sim_f32_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int Na, int Nb, int d,
               long long ld) {
  __shared__ float sa[SIM_K][SIM_T + 4], sb[SIM_K][SIM_T + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int row0 = blockIdx.y * SIM_T, col0 = blockIdx.x * SIM_T;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < d; k0 += SIM_K) {
    for (int idx = threadIdx.x; idx < SIM_T * SIM_K; idx += 256) {
      const int r = idx / SIM_K, k = idx - r * SIM_K;
      sa[k][r] = (row0 + r < Na && k0 + k < d) ? a[static_cast<long long>(row0 + r) * d + k0 + k] : 0.f;
      sb[k][r] = (col0 + r < Nb && k0 + k < d) ? b[static_cast<long long>(col0 + r) * d + k0 + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SIM_K; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        av[i] = sa[k][ty * 4 + i];
        bv[i] = sb[k][tx * 4 + i];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = row0 + ty * 4 + i, c = col0 + tx * 4 + j;
      if (r < Na && c < Nb) out[static_cast<long long>(r) * ld + c] = acc[i][j];
    }
}

// Column statistics of theta * sim: max and sum of exp(. - max).  One thread per column (rows are walked coalesced
// across the 32 columns of a warp).
__global__ void __launch_bounds__(128)
dsl_colstats_kernel(const float* __restrict__ sim, int rows, int cols, long long ld, float theta, float* __restrict__ cmax,
                    float* __restrict__ csum) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= cols) return;
  float m = -INFINITY;
  for (int r = 0; r < rows; ++r) m = fmaxf(m, sim[static_cast<long long>(r) * ld + c] * theta);
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += expf(sim[static_cast<long long>(r) * ld + c] * theta - m);
  cmax[c] = m;
  csum[c] = s;
}
__global__ void __launch_bounds__(256)
dsl_apply_kernel(float* __restrict__ sim, int rows, int cols, long long ld, float theta, const float* __restrict__ cmax,
                 const float* __restrict__ csum) {
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(rows) * cols) return;
  const int r = static_cast<int>(idx / cols), c = static_cast<int>(idx - static_cast<long long>(r) * cols);
  float* p = sim + static_cast<long long>(r) * ld + c;
  const float v = *p;
  *p = v * (expf(v * theta - cmax[c]) / csum[c]);
}

// One warp per query i: entries x[i, j] (transpose: x[j, i]) compared with the diagonal x[i, i].
__global__ void __launch_bounds__(128)
rank_counts_kernel(const float* __restrict__ sim, int N, long long ld, int transpose, int* __restrict__ greater,
                   int* __restrict__ equal) {
  const int i = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= N) return;
  const float dg = sim[static_cast<long long>(i) * ld + i];
  int g = 0, e = 0;
  for (int j = lane; j < N; j += 32) {
    const float v = transpose ? sim[static_cast<long long>(j) * ld + i] : sim[static_cast<long long>(i) * ld + j];
    g += v > dg;
    e += v == dg;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    g += __shfl_xor_sync(0xffffffffu, g, o);
    e += __shfl_xor_sync(0xffffffffu, e, o);
  }
  if (lane == 0) {
    greater[i] = g;
    equal[i] = isfinite(dg) ? e : 0;   // a NaN / +-inf diagonal leaves the reference's rank list (see above)
  }
}

}  // namespace xp

using namespace xp;

extern "C" int xp_sim_f32(const float* a, const float* b, float* out, int32_t Na, int32_t Nb, int32_t d, int64_t ld,
                          void* stream) {
  XP_ENTER(a);
  if (Na <= 0 || Nb <= 0 || d <= 0 || ld < Nb) return fail("xp_sim_f32: Na, Nb, d must be positive and ld >= Nb");
  const dim3 grid((Nb + SIM_T - 1) / SIM_T, (Na + SIM_T - 1) / SIM_T);
  sim_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, b, out, Na, Nb, d, ld);
  XP_CHECK_LAUNCH("sim_f32_kernel");
  return 0;
}

extern "C" int xp_dsl_reweight(float* sim, int32_t rows, int32_t cols, int64_t ld, float theta, float* col_scratch,
                               void* stream) {
  XP_ENTER(sim);
  if (rows <= 0 || cols <= 0 || ld < cols) return fail("xp_dsl_reweight: rows, cols must be positive and ld >= cols");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dsl_colstats_kernel<<<(cols + 127) / 128, 128, 0, st>>>(sim, rows, cols, ld, theta, col_scratch, col_scratch + cols);
  XP_CHECK_LAUNCH("dsl_colstats_kernel");
  const long long n = static_cast<long long>(rows) * cols;
  dsl_apply_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(sim, rows, cols, ld, theta, col_scratch,
                                                                          col_scratch + cols);
  XP_CHECK_LAUNCH("dsl_apply_kernel");
  return 0;
}

extern "C" int xp_rank_counts(const float* sim, int32_t N, int64_t ld, int32_t transpose, int32_t* greater, int32_t* equal,
                              void* stream) {
  XP_ENTER(sim);
  if (N <= 0 || ld < N) return fail("xp_rank_counts: N must be positive and ld >= N");
  rank_counts_kernel<<<(N + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(sim, N, ld, transpose, greater, equal);
  XP_CHECK_LAUNCH("rank_counts_kernel");
  return 0;
}
