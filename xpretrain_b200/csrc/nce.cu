// The contrastive losses of loss.py around the wgmma GEMM (gemm.cu): the hi/lo split that makes the logits GEMM
// fp32-grade, and the table-driven InfoNCE family and dual-softmax loss on its fp32 logits.  NCELearnableTempLoss
// (loss.py:134-141) beyond the fused kernel's reach is the table ((rows, A), (columns, A)):
//   Z = exp(logit_scale) * V T^T                     [N, N]   (rows = videos)
//   loss = mean_i(LSE_j Z_ij - Z_ii) + mean_j(LSE_i Z_ij - Z_jj)        (SUM of the two CEs, no 1/2)
//   G = dL/dZ = (softmax_rows(Z) + softmax_cols(Z) - 2I) / N
//   dV = s G T,  dT = s G^T V,  d logit_scale = sum_ij G_ij Z_ij         (SURVEY.md §8e closed form)
//
// To keep fp32-level logits out of bf16 tensor-core inputs, V and T are split into bf16 hi + lo parts and the three
// significant cross terms are concatenated along K:  [Vh | Vh | Vl] . [Th | Tl | Th]^T  (K = 3d), i.e. one GEMM,
// ~2^-16 relative error.
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

// ---------------------------------------------------------------------------------------------------------
// Table-driven InfoNCE family (XpNceTerms, the learnable / fixed temperature losses of loss.py) and the dual-softmax
// loss (NCELearnableTempDSLLoss, loss.py:185-202).
//
// Every matrix is read in 64 x 128 tiles, row-major and coalesced: warp w holds rows 8w..8w+7, lane l holds the four
// columns 4l..4l+3 (one float4 per row).  A tile yields, for each of its rows and each of its columns, one (max, sum exp)
// partial (or a plain sum for the DSL u / w vectors); in tiles that cut the diagonal a second partial without the
// diagonal entry is kept for the terms that exclude it.  A combine kernel folds the partials of every member matrix of a
// term, in tile order, into the term's LSE vector; a gradient pass re-reads each tile and writes s * dL/dZ as bf16.
// loss and d logit_scale are reduced from per-CTA partials in a fixed order by one final CTA: no float atomics, so
// repeated calls are bit-identical.
constexpr int kTileThreads = 256, kTileRows = 64, kTileCols = 128, kRowsPerWarp = 8;
constexpr int kCombineThreads = 256;

struct NceMat {
  const float* z;            // unscaled logits [n, ld]
  __nv_bfloat16* g;          // s * dL/dZ, bf16 [n, ld]
  long long ld;
  int n, rtiles, ctiles, tile0, need_x;  // need_x: bit 0 rows, bit 1 columns have a term without the diagonal
  float2* rowp;              // [ctiles][n] row partials, one per column tile
  float2* colp;              // [rtiles][n] column partials, one per row tile
  float2* rowx;              // [n] row i in its diagonal tile, diagonal excluded
  float2* colx;              // [n] column j in its diagonal tile, diagonal excluded
};
struct NceTermDev {
  int axis, members, excl, target, n;
  float* lse;                // [n]
};
struct NcePlan {
  NceMat mat[3];
  NceTermDev term[6];
  int n_mats, n_terms, n_tiles;
  const float* logit_scale;  // device log-scale (s = exp) or NULL: s = scale
  float scale;
  float* ds_part;            // [n_tiles] per-CTA sum of G * Z
  float* loss;
  float* dscale;
  float* dsl[6];             // DSL: lse_r, lse_c, la, lb, u, w (each [n])
};

__device__ __forceinline__ float plan_scale(const NcePlan& p) { return p.logit_scale ? expf(*p.logit_scale) : p.scale; }

__device__ __forceinline__ NceMat pick_mat(const NcePlan& p, int m) { return m == 0 ? p.mat[0] : (m == 1 ? p.mat[1] : p.mat[2]); }

template <bool SUM>
__device__ __forceinline__ float2 part_merge(float2 a, float2 b) {
  if (SUM) return make_float2(a.x + b.x, 0.f);
  const float m = fmaxf(a.x, b.x);
  if (m == -INFINITY) return make_float2(-INFINITY, 0.f);
  return make_float2(m, a.y * __expf(a.x - m) + b.y * __expf(b.x - m));
}

template <bool SUM>
__device__ __forceinline__ float2 part_identity() { return SUM ? make_float2(0.f, 0.f) : make_float2(-INFINITY, 0.f); }

// The tile this CTA owns: matrix m, first row r0, first column c0.
__device__ __forceinline__ int locate_tile(const NcePlan& p, int& r0, int& c0) {
  const int b = blockIdx.x;
  const int m = (p.n_mats > 2 && b >= p.mat[2].tile0) ? 2 : ((p.n_mats > 1 && b >= p.mat[1].tile0) ? 1 : 0);
  const NceMat M = pick_mat(p, m);
  const int t = b - M.tile0;
  r0 = (t / M.ctiles) * kTileRows;
  c0 = (t % M.ctiles) * kTileCols;
  return m;
}

// x[r][k] = s * z[r0 + 8w + r][c + k]; `valid` bit (4r + k) marks entries inside the n x n matrix.
__device__ __forceinline__ unsigned load_tile(const NceMat& M, int r0, int c, float s, float (&x)[kRowsPerWarp][4]) {
  const int row0 = r0 + (threadIdx.x >> 5) * kRowsPerWarp;
  unsigned valid = 0;
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < M.n && c < M.n) v = __ldg(reinterpret_cast<const float4*>(M.z + static_cast<long long>(row0 + r) * M.ld + c));
    x[r][0] = s * v.x; x[r][1] = s * v.y; x[r][2] = s * v.z; x[r][3] = s * v.w;
    if (row0 + r < M.n) {
#pragma unroll
      for (int k = 0; k < 4; ++k) valid |= (c + k < M.n ? 1u : 0u) << (4 * r + k);
    }
  }
  return valid;
}

// Row and column partials of one tile.  rv feeds the row statistics, cv the column statistics; entries outside `valid`
// (and the diagonal when diag_only) are left out.  Rows / columns are written to rowdst[i] / coldst[j]; with diag_only
// only those whose diagonal entry lies inside the tile (the diagonal-excluded partials).
template <bool SUM>
__device__ void tile_partials(const float (&rv)[kRowsPerWarp][4], const float (&cv)[kRowsPerWarp][4], unsigned valid,
                              int r0, int c0, int n, bool diag_only, float2* rowdst, float2* coldst, float2 (*sh)[kTileCols]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = r0 + warp * kRowsPerWarp, c = c0 + 4 * lane;
  auto keep = [&](int r, int k) { return ((valid >> (4 * r + k)) & 1u) && !(diag_only && row0 + r == c + k); };
  // rows: one warp-wide reduction per row
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    const int i = row0 + r;
    const bool want = i < n && (!diag_only || (i >= c0 && i < c0 + kTileCols));   // warp-uniform
    if (!want) continue;
    float2 acc;
    if (SUM) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) t += keep(r, k) ? rv[r][k] : 0.f;
      acc = make_float2(warp_sum(t), 0.f);
    } else {
      float mx = -INFINITY;
#pragma unroll
      for (int k = 0; k < 4; ++k) mx = fmaxf(mx, keep(r, k) ? rv[r][k] : -INFINITY);
      mx = warp_max(mx);
      float t = 0.f;
      if (mx != -INFINITY) {
#pragma unroll
        for (int k = 0; k < 4; ++k) t += keep(r, k) ? __expf(rv[r][k] - mx) : 0.f;
      }
      acc = make_float2(mx, warp_sum(t));
    }
    if (lane == 0) rowdst[i] = acc;
  }
  // columns: this thread's 8 rows, then the 8 warps in order through shared memory
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float2 acc = part_identity<SUM>();
    if (SUM) {
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) acc.x += keep(r, k) ? cv[r][k] : 0.f;
    } else {
      float mx = -INFINITY;
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) mx = fmaxf(mx, keep(r, k) ? cv[r][k] : -INFINITY);
      float t = 0.f;
      if (mx != -INFINITY) {
#pragma unroll
        for (int r = 0; r < kRowsPerWarp; ++r) t += keep(r, k) ? __expf(cv[r][k] - mx) : 0.f;
      }
      acc = make_float2(mx, t);
    }
    sh[warp][4 * lane + k] = acc;
  }
  __syncthreads();
  if (threadIdx.x < kTileCols) {
    const int j = c0 + threadIdx.x;
    float2 acc = sh[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < kTileThreads / 32; ++w) acc = part_merge<SUM>(acc, sh[w][threadIdx.x]);
    if (j < n && (!diag_only || (j >= r0 && j < r0 + kTileRows))) coldst[j] = acc;
  }
  __syncthreads();
}

// MODE 0: plain logits (row and column statistics of s*z, plus the diagonal-excluded variants the terms need).
// MODE 1: DSL, rows of A' = Z * Pc and columns of B' = Z * Pr.
// MODE 2: DSL, w_i = sum_j GB Z Pr (rows) and u_j = sum_i GA Z Pc (columns), plain sums.
template <int MODE>
__global__ void __launch_bounds__(kTileThreads) nce_tile_stats_kernel(const NcePlan p) {
  __shared__ float2 sh[kTileThreads / 32][kTileCols];
  int r0, c0;
  const int m = locate_tile(p, r0, c0);
  const NceMat M = pick_mat(p, m);
  const int c = c0 + 4 * (threadIdx.x & 31), row0 = r0 + (threadIdx.x >> 5) * kRowsPerWarp;
  const float s = plan_scale(p);
  float x[kRowsPerWarp][4];
  const unsigned valid = load_tile(M, r0, c, s, x);
  float2* rowdst = M.rowp + static_cast<long long>(c0 / kTileCols) * M.n;
  float2* coldst = M.colp + static_cast<long long>(r0 / kTileRows) * M.n;
  if (MODE == 0) {
    tile_partials<false>(x, x, valid, r0, c0, M.n, false, rowdst, coldst, sh);
    if (M.need_x && r0 < c0 + kTileCols && c0 < r0 + kTileRows)
      tile_partials<false>(x, x, valid, r0, c0, M.n, true, M.rowx, M.colx, sh);
    return;
  }
  const float *lse_r = p.dsl[0], *lse_c = p.dsl[1];
  const float inv_n = 1.f / M.n;
  float rv[kRowsPerWarp][4], cv[kRowsPerWarp][4];
  float lc[4], lb[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    lc[k] = lse_c[min(c + k, M.n - 1)];
    lb[k] = MODE == 2 ? p.dsl[3][min(c + k, M.n - 1)] : 0.f;
  }
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    const int i = min(row0 + r, M.n - 1);
    const float lr = lse_r[i], la = MODE == 2 ? p.dsl[2][i] : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float z = x[r][k];
      const float pc = __expf(z - lc[k]), pr = __expf(z - lr);
      if (MODE == 1) {
        rv[r][k] = z * pc;
        cv[r][k] = z * pr;
      } else {
        const float d = (row0 + r == c + k) ? 1.f : 0.f;
        const float ga = (__expf(z * pc - la) - d) * inv_n, gb = (__expf(z * pr - lb[k]) - d) * inv_n;
        rv[r][k] = gb * z * pr;
        cv[r][k] = ga * z * pc;
      }
    }
  }
  tile_partials<MODE == 2>(rv, cv, valid, r0, c0, M.n, false, rowdst, coldst, sh);
}

// One thread per (term, index): fold the partials of every member matrix, in tile order, into the term's LSE (or sum).
template <bool SUM>
__global__ void __launch_bounds__(kCombineThreads) nce_combine_kernel(const NcePlan p) {
  const int t = blockIdx.y, i = blockIdx.x * kCombineThreads + threadIdx.x;
  NceTermDev T = p.term[0];
#pragma unroll
  for (int u = 1; u < 6; ++u)
    if (u == t) T = p.term[u];
  if (i >= T.n) return;
  float2 acc = part_identity<SUM>();
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    if (m >= p.n_mats || !((T.members >> m) & 1)) continue;
    const NceMat& M = p.mat[m];
    const bool row = T.axis == 0;
    const float2* part = row ? M.rowp : M.colp;
    const int tiles = row ? M.ctiles : M.rtiles;
    const int kd = ((T.excl >> m) & 1) ? i / (row ? kTileCols : kTileRows) : -1;
    const float2 xd = kd >= 0 ? (row ? M.rowx : M.colx)[i] : make_float2(0.f, 0.f);
    for (int k = 0; k < tiles; ++k) acc = part_merge<SUM>(acc, k == kd ? xd : part[static_cast<long long>(k) * M.n + i]);
  }
  T.lse[i] = SUM ? acc.x : acc.x + logf(acc.y);
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) t += red[w];
  return t;   // valid in thread 0
}

// MODE 0: G = sum over the terms containing the matrix of softmax / n, minus delta / n per term targeting it.
// MODE 1: DSL, G_Z = Pc (GA (1 + Z) - u_j) + Pr (GB (1 + Z) - w_i).
// Writes s * G as bf16 (one 8-byte store per row and thread) and this CTA's sum of G * Z to ds_part.
template <int MODE>
__global__ void __launch_bounds__(kTileThreads) nce_tile_grad_kernel(const NcePlan p) {
  __shared__ float red[kTileThreads / 32];
  int r0, c0;
  const int m = locate_tile(p, r0, c0);
  const NceMat M = pick_mat(p, m);
  const int c = c0 + 4 * (threadIdx.x & 31), row0 = r0 + (threadIdx.x >> 5) * kRowsPerWarp;
  const float s = plan_scale(p);
  float x[kRowsPerWarp][4];
  const unsigned valid = load_tile(M, r0, c, s, x);
  const float inv_n = 1.f / M.n;
  float acc = 0.f;
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    const int i = row0 + r;
    if (i >= M.n || c >= M.n) continue;
    float g[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = min(c + k, M.n - 1);
      const float z = x[r][k];
      const float d = (i == c + k) ? 1.f : 0.f;
      float gg = 0.f;
      if (MODE == 0) {
#pragma unroll
        for (int t = 0; t < 6; ++t) {
          const NceTermDev& T = p.term[t];
          if (t >= p.n_terms) break;
          if (!((T.members >> m) & 1)) continue;
          if (!(((T.excl >> m) & 1) && d != 0.f)) gg += __expf(z - T.lse[T.axis == 0 ? i : j]);
          if (T.target == m) gg -= d;
        }
        gg *= inv_n;     // every term containing this matrix has its n
      } else {
        const float pc = __expf(z - p.dsl[1][j]), pr = __expf(z - p.dsl[0][i]);
        const float ga = (__expf(z * pc - p.dsl[2][i]) - d) * inv_n, gb = (__expf(z * pr - p.dsl[3][j]) - d) * inv_n;
        gg = pc * (ga * (1.f + z) - p.dsl[4][j]) + pr * (gb * (1.f + z) - p.dsl[5][i]);
      }
      const bool in = (valid >> (4 * r + k)) & 1u;
      g[k] = in ? gg : 0.f;
      acc += in ? gg * z : 0.f;
    }
    __align__(8) __nv_bfloat162 v[2] = {__floats2bfloat162_rn(g[0] * s, g[1] * s), __floats2bfloat162_rn(g[2] * s, g[3] * s)};
    *reinterpret_cast<uint2*>(M.g + static_cast<long long>(i) * M.ld + c) = *reinterpret_cast<const uint2*>(v);
  }
  const float t = block_sum(acc, red);
  if (threadIdx.x == 0) p.ds_part[blockIdx.x] = t;
}

// One CTA: loss = sum_t mean_i (LSE_t[i] - target_ii) (MODE 0) or the two DSL cross-entropies (MODE 1), and
// d logit_scale = sum of the per-tile G * Z partials, both in a fixed order.
template <int MODE>
__global__ void __launch_bounds__(kTileThreads) nce_final_kernel(const NcePlan p) {
  __shared__ float red[kTileThreads / 32];
  const float s = plan_scale(p);
  float ds = 0.f, l = 0.f;
  for (int k = threadIdx.x; k < p.n_tiles; k += blockDim.x) ds += p.ds_part[k];
  if (MODE == 0) {
#pragma unroll
    for (int t = 0; t < 6; ++t) {
      if (t >= p.n_terms) break;
      const NceTermDev& T = p.term[t];
      const NceMat M = pick_mat(p, T.target);
      float lt = 0.f;
      for (int i = threadIdx.x; i < T.n; i += blockDim.x) lt += T.lse[i] - s * M.z[static_cast<long long>(i) * M.ld + i];
      l += lt / T.n;
    }
  } else {
    const NceMat& M = p.mat[0];
    for (int i = threadIdx.x; i < M.n; i += blockDim.x) {
      const float z = s * M.z[static_cast<long long>(i) * M.ld + i];
      l += p.dsl[2][i] - z * __expf(z - p.dsl[1][i]) + p.dsl[3][i] - z * __expf(z - p.dsl[0][i]);
    }
    l /= M.n;
  }
  const float lsum = block_sum(l, red);
  const float dsum = block_sum(ds, red);
  if (threadIdx.x == 0) {
    *p.loss = lsum;
    if (p.logit_scale && p.dscale) *p.dscale = dsum;
  }
}

}  // namespace xp

using namespace xp;

namespace {

constexpr long long align4(long long v) { return (v + 3) / 4 * 4; }

// Workspace layout shared by xp_nce_terms and xp_nce_dsl, in floats.  With `p` and `ws` set, also fills the plan's
// pointers and tile geometry.
long long nce_layout(int n_mats, const int32_t* n, NcePlan* p, float* ws) {
  long long off = 0, nmax = 0;
  int tiles = 0;
  for (int m = 0; m < n_mats; ++m) {
    const long long nm = n[m];
    const int rt = static_cast<int>((nm + kTileRows - 1) / kTileRows), ct = static_cast<int>((nm + kTileCols - 1) / kTileCols);
    if (p) {
      NceMat& M = p->mat[m];
      M.n = n[m];
      M.rtiles = rt;
      M.ctiles = ct;
      M.tile0 = tiles;
      M.rowp = reinterpret_cast<float2*>(ws + off);
      M.colp = reinterpret_cast<float2*>(ws + off + align4(2 * ct * nm));
      M.rowx = reinterpret_cast<float2*>(ws + off + align4(2 * ct * nm) + align4(2 * rt * nm));
      M.colx = M.rowx + nm;
    }
    off += align4(2 * ct * nm) + align4(2 * rt * nm) + align4(4 * nm);
    tiles += rt * ct;
    nmax = nm > nmax ? nm : nmax;
  }
  if (p) {
    for (int t = 0; t < 6; ++t) p->term[t].lse = p->dsl[t] = ws + off + t * align4(nmax);
    p->ds_part = ws + off + 6 * align4(nmax);
    p->n_mats = n_mats;
    p->n_tiles = tiles;
  }
  return off + 6 * align4(nmax) + align4(tiles);
}

int nce_check_matrix(const char* who, const float* z, const void* g, int64_t ld, int32_t n) {
  if (n <= 0) return fail(std::string(who) + ": every matrix needs n > 0");
  if (!z || !g) return fail(std::string(who) + ": logits and gradient pointers are required");
  if (ld < n || ld % 4 != 0) return fail(std::string(who) + ": the row pitch must be >= n and a multiple of 4");
  if (reinterpret_cast<uintptr_t>(z) % 16 != 0 || reinterpret_cast<uintptr_t>(g) % 8 != 0)
    return fail(std::string(who) + ": logits must be 16-byte and gradients 8-byte aligned");
  return 0;
}

}  // namespace

extern "C" int64_t xp_nce_terms_workspace_bytes(const XpNceTerms* a) {
  if (!a || a->n_mats < 1 || a->n_mats > 3) return -1;
  for (int m = 0; m < a->n_mats; ++m)
    if (a->n[m] <= 0) return -1;
  return 4 * nce_layout(a->n_mats, a->n, nullptr, nullptr);
}

extern "C" int64_t xp_nce_dsl_workspace_bytes(int32_t n) {
  if (n <= 0) return -1;
  return 4 * nce_layout(1, &n, nullptr, nullptr);
}

extern "C" int xp_nce_terms(const XpNceTerms* a, void* stream) {
  if (!a) return fail("xp_nce_terms: null descriptor");
  XP_ENTER(a->z[0]);
  if (a->n_mats < 1 || a->n_mats > 3) return fail("xp_nce_terms: n_mats must be 1..3");
  if (a->n_terms < 1 || a->n_terms > 6) return fail("xp_nce_terms: n_terms must be 1..6");
  if (!a->loss || !a->workspace) return fail("xp_nce_terms: loss and workspace are required");
  if (!a->logit_scale && !(a->scale > 0.f)) return fail("xp_nce_terms: without logit_scale the host scale must be > 0");
  for (int m = 0; m < a->n_mats; ++m)
    if (nce_check_matrix("xp_nce_terms", a->z[m], a->g[m], a->ld[m], a->n[m])) return -1;
  NcePlan p{};
  nce_layout(a->n_mats, a->n, &p, a->workspace);
  const int all = (1 << a->n_mats) - 1;
  for (int t = 0; t < a->n_terms; ++t) {
    const XpNceTerm& T = a->term[t];
    const std::string at = "xp_nce_terms: term " + std::to_string(t) + ": ";
    if (T.axis != 0 && T.axis != 1) return fail(at + "axis must be 0 (rows) or 1 (columns)");
    if (T.members == 0 || (T.members & ~all)) return fail(at + "members must name existing matrices");
    if (T.excl_diag & ~T.members) return fail(at + "excl_diag must be a subset of members");
    if (T.target < 0 || T.target >= a->n_mats || !((T.members >> T.target) & 1))
      return fail(at + "the target must be a member");
    if ((T.excl_diag >> T.target) & 1) return fail(at + "the target's diagonal cannot be excluded");
    int n = -1;
    for (int m = 0; m < a->n_mats; ++m) {
      if (!((T.members >> m) & 1)) continue;
      if (n >= 0 && a->n[m] != n) return fail(at + "a union of matrices needs one n");
      n = a->n[m];
    }
    p.term[t].axis = T.axis;
    p.term[t].members = T.members;
    p.term[t].excl = T.excl_diag;
    p.term[t].target = T.target;
    p.term[t].n = n;
    for (int m = 0; m < a->n_mats; ++m)
      if ((T.excl_diag >> m) & 1) p.mat[m].need_x |= T.axis == 0 ? 1 : 2;
  }
  for (int m = 0; m < a->n_mats; ++m) {
    p.mat[m].z = a->z[m];
    p.mat[m].g = static_cast<__nv_bfloat16*>(a->g[m]);
    p.mat[m].ld = a->ld[m];
  }
  p.n_terms = a->n_terms;
  p.logit_scale = a->logit_scale;
  p.scale = a->scale;
  p.loss = a->loss;
  p.dscale = a->d_logit_scale;
  int nmax = 0;
  for (int m = 0; m < a->n_mats; ++m) nmax = a->n[m] > nmax ? a->n[m] : nmax;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  nce_tile_stats_kernel<0><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_stats_kernel");
  nce_combine_kernel<false><<<dim3((nmax + kCombineThreads - 1) / kCombineThreads, p.n_terms), kCombineThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_combine_kernel");
  nce_tile_grad_kernel<0><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_grad_kernel");
  nce_final_kernel<0><<<1, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_final_kernel");
  return 0;
}

extern "C" int xp_nce_dsl(const float* z, int64_t ld, int32_t n, const float* logit_scale, void* g_bf16, float* loss,
                          float* d_logit_scale, float* workspace, void* stream) {
  XP_ENTER(z);
  if (nce_check_matrix("xp_nce_dsl", z, g_bf16, ld, n)) return -1;
  if (!logit_scale || !loss || !workspace) return fail("xp_nce_dsl: logit_scale, loss and workspace are required");
  NcePlan p{};
  nce_layout(1, &n, &p, workspace);
  p.mat[0].z = z;
  p.mat[0].g = static_cast<__nv_bfloat16*>(g_bf16);
  p.mat[0].ld = ld;
  p.logit_scale = logit_scale;
  p.loss = loss;
  p.dscale = d_logit_scale;
  p.n_terms = 2;
  for (int t = 0; t < 2; ++t) {
    p.term[t].axis = t;
    p.term[t].members = 1;
    p.term[t].n = n;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 cgrid((n + kCombineThreads - 1) / kCombineThreads, 2);
  // 1. row / column LSE of Z
  p.term[0].lse = p.dsl[0];
  p.term[1].lse = p.dsl[1];
  nce_tile_stats_kernel<0><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_stats_kernel");
  nce_combine_kernel<false><<<cgrid, kCombineThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_combine_kernel");
  // 2. row LSE of A' = Z Pc, column LSE of B' = Z Pr
  p.term[0].lse = p.dsl[2];
  p.term[1].lse = p.dsl[3];
  nce_tile_stats_kernel<1><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_stats_kernel");
  nce_combine_kernel<false><<<cgrid, kCombineThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_combine_kernel");
  // 3. w (row sums) and u (column sums)
  p.term[0].lse = p.dsl[5];
  p.term[1].lse = p.dsl[4];
  nce_tile_stats_kernel<2><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_stats_kernel");
  nce_combine_kernel<true><<<cgrid, kCombineThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_combine_kernel");
  // 4. G_Z, loss, d logit_scale
  nce_tile_grad_kernel<1><<<p.n_tiles, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_tile_grad_kernel");
  nce_final_kernel<1><<<1, kTileThreads, 0, st>>>(p);
  XP_CHECK_LAUNCH("nce_final_kernel");
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
