// HBM-bound row kernels of the CLIP-ViP path: LayerNorm forward/backward (with the residual-gradient
// add fused), L2 normalisation forward/backward, bias-gradient column sums, fp32->bf16 parameter casts.
// One warp per row, 16-byte vector accesses, fp32 statistics.
//
// Reference ops replaced: nn.LayerNorm at CLIP_ViP.py:447,458 (layer_norm1/2), :881 (pre_layrnorm),
// :892 (post_layernorm), :771 (final_layer_norm); `x / x.norm(dim=-1, keepdim=True)` at :1148-1149.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

struct RowMapDev {
  long long group, group_stride, ld;
  const long long* offsets;  // optional explicit element offset per row
};
__device__ __forceinline__ long long row_addr(const RowMapDev& m, long long r) {
  if (m.offsets) return m.offsets[r];
  if (m.group > 0) return (r / m.group) * m.group_stride + (r % m.group) * m.ld;
  return r * m.ld;
}
static RowMapDev to_dev(const XpRowMap& m) {
  RowMapDev d;
  d.group = m.group;
  d.group_stride = m.group_stride;
  d.ld = m.ld;
  d.offsets = reinterpret_cast<const long long*>(m.offsets);
  return d;
}

constexpr int LN_MAX_VEC = 4;  // C <= 4 * 32 * 8 = 1024

// ------------------------------------------------------------------ LayerNorm forward
// Optionally fused with the residual add in fp32 (the reference keeps the residual stream in fp32 under autocast; a bf16
// stream multiplies its feature error):  s = x (+ add);  sum_out = s (fp32);
// y = LN(s).  XT / YT are the element types of x and y: bf16, fp32, or fp16 (the residual stream may be kept in fp32,
// or in fp16 as under the reference's apex O2); add is the bf16 branch output (ADD).
template <class XT, class YT, bool ADD>
__global__ void __launch_bounds__(128)
ln_fwd_kernel(const void* __restrict__ x, RowMapDev xm, const __nv_bfloat16* __restrict__ add, RowMapDev am,
              void* __restrict__ sum_out, RowMapDev sm, void* __restrict__ y, RowMapDev ym,
              const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, long long rows, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const long long r = static_cast<long long>(blockIdx.x) * 4 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int nvec = C >> 3;
  const long long xo = row_addr(xm, r);
  const long long ao = ADD ? row_addr(am, r) : 0;
  const long long so = (ADD && sum_out) ? row_addr(sm, r) : 0;
  float v[LN_MAX_VEC][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      if constexpr (std::is_same_v<XT, __half>)
        unpack8_f16(*reinterpret_cast<const uint4*>(static_cast<const __half*>(x) + xo + c * 8), v[i]);
      else
        load8(static_cast<const XT*>(x) + xo + c * 8, v[i]);
      if (ADD) {
        float a[8];
        load8(add + ao + c * 8, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] += a[j];
        if constexpr (std::is_same_v<XT, __half>) {   // fp16 stream: normalise exactly the rounded values that are stored / read back later
          const uint4 hv = pack8_f16_satfinite(v[i]);
          unpack8_f16(hv, v[i]);
          if (sum_out) *reinterpret_cast<uint4*>(static_cast<__half*>(sum_out) + so + c * 8) = hv;
        } else if (sum_out) {                // bf16 / fp32 x: the stream is stored in fp32
          store8(static_cast<float*>(sum_out) + so + c * 8, v[i]);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[i][j] - mean;
        q += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  const long long yo = row_addr(ym, r);
#pragma unroll
  for (int i = 0; i < LN_MAX_VEC; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
      const float4 g0 = *reinterpret_cast<const float4*>(gamma + c * 8), g1 = *reinterpret_cast<const float4*>(gamma + c * 8 + 4);
      const float4 b0 = *reinterpret_cast<const float4*>(beta + c * 8), b1 = *reinterpret_cast<const float4*>(beta + c * 8 + 4);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * gg[j] + bb[j];
      if constexpr (std::is_same_v<YT, __half>) store8_satfinite(static_cast<__half*>(y) + yo + c * 8, o);
      else store8(static_cast<YT*>(y) + yo + c * 8, o);
    }
  }
  if (lane == 0) {
    if (mean_out) mean_out[r] = mean;
    if (rstd_out) rstd_out[r] = rstd;
  }
}

// ----------------------------------------------------------------- LayerNorm backward
// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ dres), g = dy * gamma;
// dgamma += sum_rows dy * xhat, dbeta += sum_rows dy  (fp32 atomics, one per column per CTA).
constexpr int LNB_WARPS = 8;
// RSUM: additionally accumulate the column sums of dres into dres_sum — dres is the gradient of a residual add whose other
// branch ends in a Linear, so its column sum IS that Linear's bias gradient (fc2.bias from LN2's dres, out_proj.bias from
// LN1's): the pass that already streams dres produces it, and the standalone colsum launches disappear.
template <int NVEC, bool RSUM, class XT>
__global__ void __launch_bounds__(LNB_WARPS * 32, 2)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, RowMapDev dym, const void* __restrict__ x, RowMapDev xm,
              const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
              const __nv_bfloat16* __restrict__ dres, RowMapDev drm, __nv_bfloat16* __restrict__ dx, RowMapDev dxm,
              float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dres_sum, long long rows, int C) {
  constexpr int NACC = RSUM ? 3 : 2;
  extern __shared__ float red[];  // [LNB_WARPS][NACC][C], gamma staged behind it
  float* sgamma = red + LNB_WARPS * NACC * C;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = C >> 3;
  for (int c = threadIdx.x; c < C; c += blockDim.x) sgamma[c] = gamma[c];
  __syncthreads();
  float ag[NVEC][8], ab[NVEC][8], ar[RSUM ? NVEC : 1][8];
#pragma unroll
  for (int i = 0; i < NVEC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      ag[i][j] = ab[i][j] = 0.f;
      if (RSUM) ar[i][j] = 0.f;
    }
  for (long long r = static_cast<long long>(blockIdx.x) * LNB_WARPS + warp; r < rows;
       r += static_cast<long long>(gridDim.x) * LNB_WARPS) {
    const long long xo = row_addr(xm, r);
    const __nv_bfloat16* dyr = dy + row_addr(dym, r);
    const __nv_bfloat16* drr = dres ? dres + row_addr(drm, r) : nullptr;
    const float mu = mean[r], rs = rstd[r];
    constexpr bool XF32 = std::is_same_v<XT, float>;
    uint4 xraw[XF32 ? 1 : NVEC], draw[NVEC], rraw[NVEC];     // an fp32 x is re-read (L1) in the second pass, not kept
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        if (!XF32) xraw[i] = *reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(x) + xo + c * 8);
        draw[i] = *reinterpret_cast<const uint4*>(dyr + c * 8);
        if (drr) rraw[i] = *reinterpret_cast<const uint4*>(drr + c * 8);
      }
    }
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float xv[8], dv[8];
        if (XF32) load8(static_cast<const float*>(x) + xo + c * 8, xv);
        else if (std::is_same_v<XT, __half>) unpack8_f16(xraw[i], xv);
        else unpack8_bf16(xraw[i], xv);
        unpack8_bf16(draw[i], dv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xv[j] - mu) * rs;
          const float g = dv[j] * sgamma[c * 8 + j];
          s1 += g;
          s2 += g * xh;
          ag[i][j] += dv[j] * xh;
          ab[i][j] += dv[j];
        }
      }
    }
    s1 = warp_sum(s1) / C;
    s2 = warp_sum(s2) / C;
    __nv_bfloat16* dxr = dx + row_addr(dxm, r);
#pragma unroll
    for (int i = 0; i < NVEC; ++i) {
      const int c = lane + i * 32;
      if (c < nvec) {
        float xv[8], dv[8], o[8];
        if (XF32) load8(static_cast<const float*>(x) + xo + c * 8, xv);
        else if (std::is_same_v<XT, __half>) unpack8_f16(xraw[i], xv);
        else unpack8_bf16(xraw[i], xv);
        unpack8_bf16(draw[i], dv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (xv[j] - mu) * rs;
          o[j] = rs * (dv[j] * sgamma[c * 8 + j] - s1 - xh * s2);
        }
        if (drr) {
          float rv[8];
          unpack8_bf16(rraw[i], rv);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            o[j] += rv[j];
            if (RSUM) ar[i][j] += rv[j];
          }
        }
        store8(dxr + c * 8, o);
      }
    }
  }
  // block reduction of the parameter gradients
#pragma unroll
  for (int i = 0; i < NVEC; ++i) {
    const int c = lane + i * 32;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        red[(warp * NACC + 0) * C + c * 8 + j] = ag[i][j];
        red[(warp * NACC + 1) * C + c * 8 + j] = ab[i][j];
        if (RSUM) red[(warp * NACC + 2) * C + c * 8 + j] = ar[i][j];
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float sg = 0.f, sb = 0.f, sr = 0.f;
#pragma unroll
    for (int w = 0; w < LNB_WARPS; ++w) {
      sg += red[(w * NACC + 0) * C + c];
      sb += red[(w * NACC + 1) * C + c];
      if (RSUM) sr += red[(w * NACC + 2) * C + c];
    }
    atomicAdd(dgamma + c, sg);
    atomicAdd(dbeta + c, sb);
    if (RSUM) atomicAdd(dres_sum + c, sr);
  }
}

// ------------------------------------------------------------------------ L2 normalise
// y = x / ||x||  (fp32 in, fp32 out, optional bf16 copy); one warp per row.
__global__ void __launch_bounds__(128)
l2norm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, float* __restrict__ inv_norm, int rows, int C) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float v = x[static_cast<long long>(r) * C + c];
    s += v * v;
  }
  const float inv = 1.f / sqrtf(warp_sum(s));
  for (int c = lane; c < C; c += 32) y[static_cast<long long>(r) * C + c] = x[static_cast<long long>(r) * C + c] * inv;
  if (lane == 0) inv_norm[r] = inv;
}
// dx = (dy - y * (y . dy)) * inv_norm, written as bf16 (it feeds the projection dgrad/wgrad GEMMs).
__global__ void __launch_bounds__(128)
l2norm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ inv_norm,
                  __nv_bfloat16* __restrict__ dx, int rows, int C, float scale) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r >= rows) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += dy[static_cast<long long>(r) * C + c] * y[static_cast<long long>(r) * C + c];
  s = warp_sum(s);
  const float inv = inv_norm[r] * scale;
  for (int c = lane; c < C; c += 32) {
    const long long i = static_cast<long long>(r) * C + c;
    dx[i] = __float2bfloat16((dy[i] - y[i] * s) * inv);
  }
}

// ------------------------------------------------------------------------ frame-mean head
// The per-frame CLIP model's video feature (VidCLIP.py:62-65), per video b over its T frame projections p_t [P]:
//   u_t = p_t / ||p_t||,  m = mean_t u_t,  f = m / ||m||          (fp32)
// One CTA per video.  Every reduction runs in a fixed order and nothing is accumulated atomically, so two calls give
// bitwise-equal results.  A zero-norm row gives inf / NaN, as the reference's division does.
constexpr int FP_THREADS = 256, FP_WARPS = FP_THREADS / 32;

// Sum of v over the CTA, the same value in every thread; warp partials are added in warp order.
__device__ __forceinline__ float frame_pool_block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < FP_WARPS; ++w) s += red[w];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(FP_THREADS)
frame_pool_fwd_kernel(const float* __restrict__ proj, float* __restrict__ feat, float* __restrict__ inv_frame,
                      float* __restrict__ inv_video, int T, int P) {
  extern __shared__ float fp_smem[];      // inverse frame norms [T] | frame mean [P]
  __shared__ float red[FP_WARPS];
  float* s_inv = fp_smem;
  float* s_m = fp_smem + T;
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* pb = proj + static_cast<long long>(b) * T * P;
  for (int t = warp; t < T; t += FP_WARPS) {          // one warp per frame
    const float* p = pb + static_cast<long long>(t) * P;
    float s = 0.f;
    for (int c = lane; c < P; c += 32) s += p[c] * p[c];
    const float inv = 1.f / sqrtf(warp_sum(s));
    if (lane == 0) {
      s_inv[t] = inv;
      inv_frame[static_cast<long long>(b) * T + t] = inv;
    }
  }
  __syncthreads();
  float ss = 0.f;
  for (int c = threadIdx.x; c < P; c += FP_THREADS) {
    float acc = 0.f;
    for (int t = 0; t < T; ++t) acc += pb[static_cast<long long>(t) * P + c] * s_inv[t];
    const float m = acc / static_cast<float>(T);
    s_m[c] = m;                                        // read back below by the same thread
    ss += m * m;
  }
  const float inv2 = 1.f / sqrtf(frame_pool_block_sum(ss, red));
  for (int c = threadIdx.x; c < P; c += FP_THREADS) feat[static_cast<long long>(b) * P + c] = s_m[c] * inv2;
  if (threadIdx.x == 0) inv_video[b] = inv2;
}

// Exact backward through both normalisations, times `scale`, written as bf16 (it feeds the projection GEMMs):
//   du = (df - f (f . df)) / (||m|| T)   (the same for every frame),   dp_t = (du - u_t (u_t . du)) / ||p_t||
// u_t is rebuilt as p_t * inv_frame[t], the product the forward formed.
__global__ void __launch_bounds__(FP_THREADS)
frame_pool_bwd_kernel(const float* __restrict__ dfeat, const float* __restrict__ feat, const float* __restrict__ proj,
                      const float* __restrict__ inv_frame, const float* __restrict__ inv_video,
                      __nv_bfloat16* __restrict__ dproj, int T, int P, float scale) {
  extern __shared__ float fp_smem[];      // du [P]
  __shared__ float red[FP_WARPS];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* df = dfeat + static_cast<long long>(b) * P;
  const float* f = feat + static_cast<long long>(b) * P;
  float s = 0.f;
  for (int c = threadIdx.x; c < P; c += FP_THREADS) s += df[c] * f[c];
  const float dot = frame_pool_block_sum(s, red);
  const float k = inv_video[b] * scale / static_cast<float>(T);
  for (int c = threadIdx.x; c < P; c += FP_THREADS) fp_smem[c] = (df[c] - f[c] * dot) * k;
  __syncthreads();
  for (int t = warp; t < T; t += FP_WARPS) {          // one warp per frame
    const long long r = static_cast<long long>(b) * T + t;
    const float* p = proj + r * P;
    const float inv = inv_frame[r];
    float d = 0.f;
    for (int c = lane; c < P; c += 32) d += p[c] * inv * fp_smem[c];
    d = warp_sum(d);
    for (int c = lane; c < P; c += 32) dproj[r * P + c] = __float2bfloat16((fp_smem[c] - p[c] * inv * d) * inv);
  }
}

// ------------------------------------------------------------------------- column sums
// out[c] += sum_r x[r, c]   (bias gradients).  grid.x covers column chunks of 256, grid.y splits rows.
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, long long ld, float* __restrict__ out, long long rows, int C,
              float scale) {
  __shared__ float part[8][256];
  const int col8 = threadIdx.x & 31;        // 32 lanes x 8 columns = 256 columns
  const int rl = threadIdx.x >> 5;          // 8 row lanes
  const int c0 = blockIdx.x * 256 + col8 * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c0 < C) {
    for (long long r = static_cast<long long>(blockIdx.y) * 8 + rl; r < rows; r += static_cast<long long>(gridDim.y) * 8) {
      float v[8];
      load8(x + r * ld + c0, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) part[rl][col8 * 8 + j] = acc[j];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < C) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += part[w][threadIdx.x];
    atomicAdd(out + c, s * scale);
  }
}

// ------------------------------------------------------------------ fp32 -> bf16 casts
__global__ void __launch_bounds__(256)
cast_f32_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  const long long i = (static_cast<long long>(blockIdx.x) * 256 + threadIdx.x) * 8;
  if (i + 8 <= n) {
    float f[8];
    load8(src + i, f);
    store8(dst + i, f);
  } else {
    for (long long j = i; j < n; ++j) dst[j] = __float2bfloat16(src[j]);
  }
}

// ------------------------------------------------- per-row scale (+ residual): stochastic depth
// out[r, :] = (res ? res[r, :] : 0) + scale[r] * x[r, :]   — DropPath of timesformer.py:98-113 applied to a residual
// branch: scale[r] is 0 or 1/keep_prob for the sample (or group) row r belongs to.  One thread per 8 columns.
__global__ void __launch_bounds__(256)
rowscale_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ scale, const __nv_bfloat16* __restrict__ res,
                __nv_bfloat16* __restrict__ out, long long rows, int C) {
  const int vec = C >> 3;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= rows * vec) return;
  const long long r = idx / vec;
  const long long off = r * C + (idx - r * vec) * 8;
  const float s = scale[r];
  float v[8];
  load8(x + off, v);
  if (res != nullptr) {
    float q[8];
    load8(res + off, q);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = q[j] + s * v[j];
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= s;
  }
  store8(out + off, v);
}

// ------------------------------------------------- LayerNorm over rows wider than 1024 columns
// PatchMerging's LayerNorm(4C) of LF-VILA's Swin-3D reaches 2048 columns (video_encoder.py:281,304).  One CTA of 256
// threads per row; thread t owns columns {t*8 + k*2048}.  Rows are contiguous (ld = C).  Rarely on the critical path
// (three launches per forward), so it favours simplicity: the row is read twice (mean, then centred variance).
constexpr int LNW_THREADS = 256;
constexpr int LNW_MAXK = 2;            // C <= 2 * 2048
__device__ __forceinline__ float block_sum256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                     // protects `red` against the previous use
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < LNW_THREADS / 32; ++w) s += red[w];
  return s;
}
__global__ void __launch_bounds__(LNW_THREADS)
ln_wide_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, const float* __restrict__ gamma,
                   const float* __restrict__ beta, float* __restrict__ mean_out, float* __restrict__ rstd_out, int C,
                   float eps) {
  __shared__ float red[LNW_THREADS / 32];
  const long long r = blockIdx.x;
  const __nv_bfloat16* xr = x + r * C;
  float v[LNW_MAXK][8];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < LNW_MAXK; ++k) {
    const int c = threadIdx.x * 8 + k * LNW_THREADS * 8;
    if (c < C) {
      load8(xr + c, v[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[k][j];
    }
  }
  const float mean = block_sum256(s, red) / C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < LNW_MAXK; ++k)
    if (threadIdx.x * 8 + k * LNW_THREADS * 8 < C) {
#pragma unroll
      for (int j = 0; j < 8; ++j) q += (v[k][j] - mean) * (v[k][j] - mean);
    }
  const float rstd = rsqrtf(block_sum256(q, red) / C + eps);
#pragma unroll
  for (int k = 0; k < LNW_MAXK; ++k) {
    const int c = threadIdx.x * 8 + k * LNW_THREADS * 8;
    if (c < C) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[k][j] - mean) * rstd * gamma[c + j] + beta[c + j];
      store8(y + r * C + c, o);
    }
  }
  if (threadIdx.x == 0) {
    mean_out[r] = mean;
    rstd_out[r] = rstd;
  }
}
// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma; dgamma += dy * xhat, dbeta += dy.  Each CTA walks
// rows blockIdx.x, blockIdx.x + gridDim.x, ... keeping its column partials of dgamma / dbeta in registers.
__global__ void __launch_bounds__(LNW_THREADS)
ln_wide_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma,
                   const float* __restrict__ mean, const float* __restrict__ rstd, __nv_bfloat16* __restrict__ dx,
                   float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C) {
  __shared__ float red[LNW_THREADS / 32];
  float ag[LNW_MAXK][8] = {}, ab[LNW_MAXK][8] = {};
  for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
    const float mu = mean[r], rs = rstd[r];
    float g[LNW_MAXK][8], xh[LNW_MAXK][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < LNW_MAXK; ++k) {
      const int c = threadIdx.x * 8 + k * LNW_THREADS * 8;
      if (c < C) {
        float d[8], xv[8];
        load8(dy + r * C + c, d);
        load8(x + r * C + c, xv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[k][j] = (xv[j] - mu) * rs;
          g[k][j] = d[j] * gamma[c + j];
          s1 += g[k][j];
          s2 += g[k][j] * xh[k][j];
          ag[k][j] += d[j] * xh[k][j];
          ab[k][j] += d[j];
        }
      }
    }
    const float m1 = block_sum256(s1, red) / C;
    const float m2 = block_sum256(s2, red) / C;
#pragma unroll
    for (int k = 0; k < LNW_MAXK; ++k) {
      const int c = threadIdx.x * 8 + k * LNW_THREADS * 8;
      if (c < C) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rs * (g[k][j] - m1 - xh[k][j] * m2);
        store8(dx + r * C + c, o);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < LNW_MAXK; ++k) {
    const int c = threadIdx.x * 8 + k * LNW_THREADS * 8;
    if (c < C) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        atomicAdd(dgamma + c + j, ag[k][j]);
        atomicAdd(dbeta + c + j, ab[k][j]);
      }
    }
  }
}

// ------------------------------------------------- row gather / scatter by an index table
// out[r, k*C : (k+1)*C] = src[idx[r*segs + k], :] (zeros when the index is negative): PatchMerging's 2x2 neighbour
// concatenation with its odd-size zero padding (video_encoder.py:292-301); scatter is the exact inverse (its backward).
__global__ void __launch_bounds__(256)
gather_rows_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ idx, __nv_bfloat16* __restrict__ out,
                   long long n_items, int C) {
  const int vec = C >> 3;
  const long long gid = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (gid >= n_items * vec) return;
  const long long item = gid / vec;
  const int c = static_cast<int>(gid - item * vec) * 8;
  const int s = idx[item];
  uint4 v = make_uint4(0, 0, 0, 0);
  if (s >= 0) v = *reinterpret_cast<const uint4*>(src + static_cast<long long>(s) * C + c);
  *reinterpret_cast<uint4*>(out + item * C + c) = v;
}
__global__ void __launch_bounds__(256)
scatter_rows_kernel(const __nv_bfloat16* __restrict__ in, const int* __restrict__ idx, __nv_bfloat16* __restrict__ dst,
                    long long n_items, int C) {
  const int vec = C >> 3;
  const long long gid = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (gid >= n_items * vec) return;
  const long long item = gid / vec;
  const int c = static_cast<int>(gid - item * vec) * 8;
  const int s = idx[item];
  if (s >= 0) *reinterpret_cast<uint4*>(dst + static_cast<long long>(s) * C + c) = *reinterpret_cast<const uint4*>(in + item * C + c);
}

}  // namespace xp

using namespace xp;

// Alignment refusals for the operands the kernels above move as 16-byte vectors (uint4 / float4 / load8 / store8).
// Pure argument checks: every entry point runs them before XP_ENTER, so no misaligned operand reaches a launch.
static bool misaligned(const char* fn, const char* name, const void* p, int& rc) {
  if (aligned(p, 16)) return false;                      // NULL passes: optional operands
  rc = fail(std::string(fn) + ": " + name + " must be 16-byte aligned");
  return true;
}
// A row map's explicit offsets are device data (documented in the header); ld and group_stride are checked here.
static bool misaligned_rows(const char* fn, const char* name, const void* p, const XpRowMap* m, int elsize, int& rc) {
  if (misaligned(fn, name, p, rc)) return true;
  if (p == nullptr || m == nullptr || m->offsets != nullptr) return false;   // a map without its operand is never read
  if ((m->ld * elsize) % 16 == 0 && (m->group <= 0 || (m->group_stride * elsize) % 16 == 0)) return false;
  rc = fail(std::string(fn) + ": " + name + " rows must be 16-byte aligned (ld and group_stride times the element size "
            "must be multiples of 16 bytes)");
  return true;
}
static int dtype_bytes(int32_t dtype) { return dtype == XP_DTYPE_F32 ? 4 : 2; }

extern "C" int xp_layernorm_wide_fwd(const void* x, void* y, const float* gamma, const float* beta, float* mean, float* rstd,
                                     int64_t rows, int32_t C, float eps, void* stream) {
  const char* fn = "xp_layernorm_wide_fwd";
  if (C % 8 || C > LNW_MAXK * LNW_THREADS * 8) return fail("xp_layernorm_wide_fwd: C must be a multiple of 8 and <= 4096");
  int rc = 0;
  if (misaligned(fn, "x", x, rc) || misaligned(fn, "y", y, rc)) return rc;
  XP_ENTER(x);
  if (rows <= 0) return 0;
  ln_wide_fwd_kernel<<<static_cast<unsigned>(rows), LNW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), gamma, beta, mean, rstd, C, eps);
  XP_CHECK_LAUNCH("ln_wide_fwd_kernel");
  return 0;
}

extern "C" int xp_layernorm_wide_bwd(const void* dy, const void* x, const float* gamma, const float* mean, const float* rstd,
                                     void* dx, float* dgamma, float* dbeta, int64_t rows, int32_t C, void* stream) {
  const char* fn = "xp_layernorm_wide_bwd";
  if (C % 8 || C > LNW_MAXK * LNW_THREADS * 8) return fail("xp_layernorm_wide_bwd: C must be a multiple of 8 and <= 4096");
  int rc = 0;
  if (misaligned(fn, "dy", dy, rc) || misaligned(fn, "x", x, rc) || misaligned(fn, "dx", dx, rc)) return rc;
  XP_ENTER(dy);
  if (rows <= 0) return 0;
  const long long cap = 2LL * sm_count();
  ln_wide_bwd_kernel<<<static_cast<unsigned>(rows < cap ? rows : cap), LNW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(dy), static_cast<const __nv_bfloat16*>(x), gamma, mean, rstd,
      static_cast<__nv_bfloat16*>(dx), dgamma, dbeta, rows, C);
  XP_CHECK_LAUNCH("ln_wide_bwd_kernel");
  return 0;
}

extern "C" int xp_gather_rows_bf16(const void* src, const int32_t* index, void* out, int64_t n_items, int32_t C, void* stream) {
  if (C % 8) return fail("xp_gather_rows_bf16: C must be a multiple of 8");
  int rc = 0;
  if (misaligned("xp_gather_rows_bf16", "src", src, rc) || misaligned("xp_gather_rows_bf16", "out", out, rc)) return rc;
  XP_ENTER(src);
  if (n_items <= 0) return 0;
  const long long n = n_items * (C / 8);
  gather_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(src), index, static_cast<__nv_bfloat16*>(out), n_items, C);
  XP_CHECK_LAUNCH("gather_rows_kernel");
  return 0;
}

extern "C" int xp_scatter_rows_bf16(const void* in, const int32_t* index, void* dst, int64_t n_items, int32_t C, void* stream) {
  if (C % 8) return fail("xp_scatter_rows_bf16: C must be a multiple of 8");
  int rc = 0;
  if (misaligned("xp_scatter_rows_bf16", "in", in, rc) || misaligned("xp_scatter_rows_bf16", "dst", dst, rc)) return rc;
  XP_ENTER(in);
  if (n_items <= 0) return 0;
  const long long n = n_items * (C / 8);
  scatter_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(in), index, static_cast<__nv_bfloat16*>(dst), n_items, C);
  XP_CHECK_LAUNCH("scatter_rows_kernel");
  return 0;
}

extern "C" int xp_rowscale_bf16(const void* x, const float* scale, const void* residual, void* out, int64_t rows, int32_t C,
                                void* stream) {
  const char* fn = "xp_rowscale_bf16";
  if (C % 8) return fail("xp_rowscale_bf16: C must be a multiple of 8");
  int rc = 0;
  if (misaligned(fn, "x", x, rc) || misaligned(fn, "residual", residual, rc) || misaligned(fn, "out", out, rc)) return rc;
  XP_ENTER(x);
  if (rows <= 0) return 0;
  const long long n = rows * (C / 8);
  rowscale_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), scale, static_cast<const __nv_bfloat16*>(residual),
      static_cast<__nv_bfloat16*>(out), rows, C);
  XP_CHECK_LAUNCH("rowscale_kernel");
  return 0;
}

extern "C" int xp_layernorm_fwd(const void* x, const XpRowMap* xmap, void* y, const XpRowMap* ymap, const float* gamma,
                                const float* beta, float* mean, float* rstd, int64_t rows, int32_t C, float eps, void* stream) {
  return xp_layernorm_add_fwd(x, xmap, XP_DTYPE_BF16, nullptr, nullptr, nullptr, nullptr, y, ymap, XP_DTYPE_BF16, gamma, beta,
                              mean, rstd, rows, C, eps, stream);
}

extern "C" int xp_layernorm_add_fwd(const void* x, const XpRowMap* xmap, int32_t x_dtype, const void* add_bf16,
                                    const XpRowMap* addmap, void* sum_out, const XpRowMap* summap, void* y,
                                    const XpRowMap* ymap, int32_t y_dtype, const float* gamma, const float* beta, float* mean,
                                    float* rstd, int64_t rows, int32_t C, float eps, void* stream) {
  if (C % 8 || C > LN_MAX_VEC * 256) return fail("xp_layernorm_fwd: C must be a multiple of 8 and <= 1024");
  const char* bad_dtype = "xp_layernorm_add_fwd: x / y dtype must be XP_DTYPE_BF16, XP_DTYPE_F32 or XP_DTYPE_F16";
  if ((x_dtype != XP_DTYPE_BF16 && x_dtype != XP_DTYPE_F32 && x_dtype != XP_DTYPE_F16) ||
      (y_dtype != XP_DTYPE_BF16 && y_dtype != XP_DTYPE_F32 && y_dtype != XP_DTYPE_F16))
    return fail(bad_dtype);
  if (add_bf16 != nullptr && addmap == nullptr) return fail("xp_layernorm_add_fwd: add needs its row map");
  if (sum_out != nullptr && (add_bf16 == nullptr || summap == nullptr)) return fail("xp_layernorm_add_fwd: sum_out needs add and its row map");
  const char* fn = "xp_layernorm_add_fwd";
  int rc = 0;
  if (misaligned_rows(fn, "x", x, xmap, dtype_bytes(x_dtype), rc) || misaligned_rows(fn, "add", add_bf16, addmap, 2, rc) ||
      misaligned_rows(fn, "sum_out", sum_out, summap, x_dtype == XP_DTYPE_F16 ? 2 : 4, rc) ||
      misaligned_rows(fn, "y", y, ymap, dtype_bytes(y_dtype), rc) || misaligned(fn, "gamma", gamma, rc) ||
      misaligned(fn, "beta", beta, rc))
    return rc;
  XP_ENTER(x);
  if (rows <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((rows + 3) / 4);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  XpRowMap none = {0, 0, 0, nullptr};
  const RowMapDev xm = to_dev(*xmap), am = to_dev(addmap ? *addmap : none), sm = to_dev(summap ? *summap : none), ym = to_dev(*ymap);
  const __nv_bfloat16* add = static_cast<const __nv_bfloat16*>(add_bf16);
  rc = dispatch_dtype(x_dtype, bad_dtype, [&](auto xt) {
    return dispatch_dtype(y_dtype, bad_dtype, [&](auto yt) {
      return dispatch<0, 1>(add != nullptr, bad_dtype, [&](auto ad) {
        ln_fwd_kernel<decltype(xt), decltype(yt), ad.value><<<grid, 128, 0, st>>>(x, xm, add, am, sum_out, sm, y, ym, gamma,
                                                                                 beta, mean, rstd, rows, C, eps);
        return 0;
      });
    });
  });
  if (rc) return rc;
  XP_CHECK_LAUNCH("ln_fwd_kernel");
  return 0;
}

extern "C" int xp_layernorm_bwd(const void* dy, const XpRowMap* dymap, const void* x, const XpRowMap* xmap, int32_t x_dtype,
                                const float* gamma, const float* mean, const float* rstd, const void* dres,
                                const XpRowMap* drmap, void* dx, const XpRowMap* dxmap, float* dgamma, float* dbeta,
                                float* dres_colsum, int64_t rows, int32_t C, void* stream) {
  const char* bad_dtype = "xp_layernorm_bwd: x dtype must be XP_DTYPE_BF16, XP_DTYPE_F32 or XP_DTYPE_F16";
  const char* bad_c = "xp_layernorm_bwd: C must be a multiple of 8 and <= 1024";
  if (x_dtype != XP_DTYPE_BF16 && x_dtype != XP_DTYPE_F32 && x_dtype != XP_DTYPE_F16) return fail(bad_dtype);
  if (C % 8 || C > LN_MAX_VEC * 256) return fail(bad_c);
  if (dres_colsum != nullptr && dres == nullptr) return fail("xp_layernorm_bwd: dres_colsum needs dres");
  const char* fn = "xp_layernorm_bwd";        // gamma is staged through shared memory element by element
  int rc = 0;
  if (misaligned_rows(fn, "dy", dy, dymap, 2, rc) || misaligned_rows(fn, "x", x, xmap, dtype_bytes(x_dtype), rc) ||
      misaligned_rows(fn, "dres", dres, drmap, 2, rc) || misaligned_rows(fn, "dx", dx, dxmap, 2, rc))
    return rc;
  XP_ENTER(dy);
  if (rows <= 0) return 0;
  long long want = (rows + LNB_WARPS - 1) / LNB_WARPS;
  const int grid = static_cast<int>(want < 4LL * sm_count() ? want : 4LL * sm_count());
  const bool rsum = dres_colsum != nullptr;
  const size_t smem = (static_cast<size_t>(LNB_WARPS) * (rsum ? 3 : 2) + 1) * C * sizeof(float);
  XpRowMap none = {0, 0, 0, nullptr};
  const int nv = (C / 8 + 31) / 32;
  rc = dispatch<1, 2, 3, 4>(nv < 1 ? 4 : nv, bad_c, [&](auto nvec) {   // C <= 0: the widest variant, no columns
    return dispatch<0, 1>(rsum, bad_c, [&](auto rs) {
      return dispatch_dtype(x_dtype, bad_dtype, [&](auto xt) {
        constexpr auto kern = ln_bwd_kernel<nvec.value, rs.value, decltype(xt)>;
        if (smem_limit<kern>((LNB_WARPS * (rs.value ? 3 : 2) + 1) * 1024 * 4)) return -1;
        kern<<<grid, LNB_WARPS * 32, smem, static_cast<cudaStream_t>(stream)>>>(
            static_cast<const __nv_bfloat16*>(dy), to_dev(*dymap), x, to_dev(*xmap), gamma, mean, rstd,
            static_cast<const __nv_bfloat16*>(dres), to_dev(drmap ? *drmap : none), static_cast<__nv_bfloat16*>(dx),
            to_dev(*dxmap), dgamma, dbeta, dres_colsum, rows, C);
        return 0;
      });
    });
  });
  if (rc) return rc;
  XP_CHECK_LAUNCH("ln_bwd_kernel");
  return 0;
}

extern "C" int xp_l2norm_fwd(const float* x, float* y, float* inv_norm, int32_t rows, int32_t C, void* stream) {
  XP_ENTER(x);
  if (rows <= 0) return 0;
  l2norm_fwd_kernel<<<(rows + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(x, y, inv_norm, rows, C);
  XP_CHECK_LAUNCH("l2norm_fwd_kernel");
  return 0;
}

extern "C" int xp_l2norm_bwd(const float* dy, const float* y, const float* inv_norm, void* dx_bf16, int32_t rows,
                             int32_t C, float scale, void* stream) {
  XP_ENTER(dy);
  if (rows <= 0) return 0;
  l2norm_bwd_kernel<<<(rows + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      dy, y, inv_norm, static_cast<__nv_bfloat16*>(dx_bf16), rows, C, scale);
  XP_CHECK_LAUNCH("l2norm_bwd_kernel");
  return 0;
}

static int frame_pool_check(const char* what, int32_t B, int32_t T, int32_t P, size_t smem) {
  if (B < 0 || T < 1 || P < 1) return fail(std::string(what) + ": need B >= 0, T >= 1 and P >= 1");
  if (B > 0x7fffffff / T) return fail(std::string(what) + ": B*T must fit in int32");
  if (smem > 48 * 1024) return fail(std::string(what) + ": T + P must be at most 12288");
  return 0;
}

extern "C" int xp_frame_pool_fwd(const float* proj, float* feat, float* inv_frame, float* inv_video, int32_t B, int32_t T,
                                 int32_t P, void* stream) {
  XP_ENTER(proj);
  const size_t smem = (static_cast<size_t>(T) + P) * sizeof(float);
  if (frame_pool_check("xp_frame_pool_fwd", B, T, P, smem)) return -1;
  if (B == 0) return 0;
  frame_pool_fwd_kernel<<<B, FP_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(proj, feat, inv_frame, inv_video, T, P);
  XP_CHECK_LAUNCH("frame_pool_fwd_kernel");
  return 0;
}

extern "C" int xp_frame_pool_bwd(const float* dfeat, const float* feat, const float* proj, const float* inv_frame,
                                 const float* inv_video, void* dproj_bf16, int32_t B, int32_t T, int32_t P, float scale,
                                 void* stream) {
  XP_ENTER(dfeat);
  const size_t smem = static_cast<size_t>(P) * sizeof(float);
  if (frame_pool_check("xp_frame_pool_bwd", B, T, P, smem)) return -1;
  if (B == 0) return 0;
  frame_pool_bwd_kernel<<<B, FP_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      dfeat, feat, proj, inv_frame, inv_video, static_cast<__nv_bfloat16*>(dproj_bf16), T, P, scale);
  XP_CHECK_LAUNCH("frame_pool_bwd_kernel");
  return 0;
}

extern "C" int xp_colsum_bf16(const void* x, int64_t ld, float* out, int64_t rows, int32_t C, float scale,
                              void* stream) {
  if (C % 8 || ld % 8) return fail("xp_colsum_bf16: C and ld must be multiples of 8");
  int rc = 0;
  if (misaligned("xp_colsum_bf16", "x", x, rc)) return rc;
  XP_ENTER(x);
  if (rows <= 0) return 0;
  const int gx = (C + 255) / 256;
  long long gy = (rows + 63) / 64;
  const long long cap = (4LL * sm_count() + gx - 1) / gx;
  if (gy > cap) gy = cap;
  colsum_kernel<<<dim3(gx, static_cast<unsigned>(gy)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), ld, out, rows, C, scale);
  XP_CHECK_LAUNCH("colsum_kernel");
  return 0;
}

extern "C" int xp_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream) {
  XP_ENTER(src);
  if (n <= 0) return 0;
  if (!aligned(src, 16) || !aligned(dst, 16))
    return fail("xp_cast_f32_bf16: pointers must be 16-byte aligned");
  const long long blocks = (n + 2047) / 2048;
  cast_f32_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      src, static_cast<__nv_bfloat16*>(dst), n);
  XP_CHECK_LAUNCH("cast_f32_bf16_kernel");
  return 0;
}
