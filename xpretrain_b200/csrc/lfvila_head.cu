// The head of LF-VILA's video classification model (LF-VILA/src/models/lfvila_video_classification.py:32-62) around the
// two projection GEMMs and the classifier GEMM:
//   pool       MaxPool2d((2, 3), stride 1) over every frame's last-stage grid, the frame mean and the clip mean
//   normalize  F.normalize(dim=-1): x / max(||x||, 1e-12)
//   ce         nn.CrossEntropyLoss (mean over the rows) and the accuracy of the first-index argmax
// Every reduction runs in a fixed order and nothing is accumulated atomically: two calls give bitwise-equal results.
// Compiled without --use_fast_math (Makefile): the means, norms and log-sum-exps use IEEE division, sqrt, exp and log.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

// ------------------------------------------------------------------------------------------------- pool
// x [B, N, Hp, Wp, C] (channels last, as the encoder returns it).  Window (i, j), i < Hp - 1, j < Wp - 2, covers rows i..i+1
// and columns j..j+2; its scan order k = kh * 3 + kw is torch's: the first maximum wins a tie, and any NaN replaces the
// running maximum (so the last NaN of the window wins), as max_pool2d's `val > max || isnan(val)`.
// CTA = 32 channels x 8 frame lanes of one clip b.  Frame lane t owns frames t, t + 8, ...; the clip sum adds the lanes'
// partial sums in lane order, so every value of the X * N window maxima enters one fp32 sum before the one division.
constexpr int POOL_FRAME_LANES = 8;

template <class T>
__global__ void __launch_bounds__(32 * POOL_FRAME_LANES)
lfvila_pool_fwd_kernel(const T* __restrict__ x, float* __restrict__ frame_raw, __nv_bfloat16* __restrict__ frame_bf16,
                       float* __restrict__ global_raw, __nv_bfloat16* __restrict__ global_bf16, uint8_t* __restrict__ argmax,
                       int N, int Hp, int Wp, int C) {
  __shared__ float part[POOL_FRAME_LANES][32];
  const int b = blockIdx.x;
  const int c = blockIdx.y * 32 + threadIdx.x;
  const int Ho = Hp - 1, Wo = Wp - 2, X = Ho * Wo;
  float gsum = 0.f;
  if (c < C) {
    for (int n = threadIdx.y; n < N; n += POOL_FRAME_LANES) {
      const long long f = static_cast<long long>(b) * N + n;
      const T* xf = x + f * Hp * Wp * C + c;
      uint8_t* am = argmax + f * X * C + c;
      float s = 0.f;
      for (int i = 0; i < Ho; ++i) {
        for (int j = 0; j < Wo; ++j) {
          float m = to_f32(xf[(static_cast<long long>(i) * Wp + j) * C]);
          int idx = 0;
#pragma unroll
          for (int k = 1; k < 6; ++k) {
            const float v = to_f32(xf[(static_cast<long long>(i + k / 3) * Wp + j + k % 3) * C]);
            if (v > m || isnan(v)) {
              m = v;
              idx = k;
            }
          }
          am[static_cast<long long>(i * Wo + j) * C] = static_cast<uint8_t>(idx);
          s += m;
        }
      }
      const float mean = s / static_cast<float>(X);
      frame_raw[f * C + c] = mean;
      frame_bf16[f * C + c] = __float2bfloat16_rn(mean);
      gsum += s;
    }
  }
  part[threadIdx.y][threadIdx.x] = gsum;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < POOL_FRAME_LANES; ++l) t += part[l][threadIdx.x];
    const float mean = t / (static_cast<float>(N) * static_cast<float>(X));
    global_raw[static_cast<long long>(b) * C + c] = mean;
    global_bf16[static_cast<long long>(b) * C + c] = __float2bfloat16_rn(mean);
  }
}

// dx[b, n, h, w, c] = (number of windows covering (h, w) whose saved arg-max is (h, w)) * g[b, n, c],
// g = d_frame[b, n, c] / X + d_global[b, c] / (N X): every window of a frame carries the same gradient (both means weigh
// its maximum equally).  A gather over the at most six covering windows: every element of dx is written, zeros included.
template <class T>
__global__ void __launch_bounds__(256)
lfvila_pool_bwd_kernel(const float* __restrict__ d_frame, const float* __restrict__ d_global, const uint8_t* __restrict__ argmax,
                       T* __restrict__ dx, long long total, int N, int Hp, int Wp, int C) {
  const int Ho = Hp - 1, Wo = Wp - 2, X = Ho * Wo;
  const long long frame_elems = static_cast<long long>(Hp) * Wp * C;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long f = e / frame_elems;
    const int rem = static_cast<int>(e - f * frame_elems);
    const int c = rem % C, pos = rem / C;
    const int h = pos / Wp, w = pos % Wp;
    const uint8_t* am = argmax + f * X * C + c;
    int cnt = 0;
    for (int i = max(0, h - 1); i <= min(h, Ho - 1); ++i)
      for (int j = max(0, w - 2); j <= min(w, Wo - 1); ++j)
        cnt += am[static_cast<long long>(i * Wo + j) * C] == (h - i) * 3 + (w - j);
    float out = 0.f;
    if (cnt) {
      float g = 0.f;
      if (d_frame) g = d_frame[f * C + c] / static_cast<float>(X);
      if (d_global) g += d_global[(f / N) * C + c] / (static_cast<float>(N) * static_cast<float>(X));
      out = static_cast<float>(cnt) * g;
    }
    dx[e] = from_f32<T>(out);
  }
}

// ------------------------------------------------------------------------------------------- normalize
// y = x / max(||x||, eps) per row (F.normalize, eps 1e-12), norm[r] = ||x|| kept for the backward.  One warp per row.
constexpr float NORM_EPS = 1e-12f;

__global__ void __launch_bounds__(128)
lfvila_normalize_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, __nv_bfloat16* __restrict__ y_bf16,
                            float* __restrict__ norm, int rows, int C) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xr = x + static_cast<long long>(r) * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c] * xr[c];
  const float n = sqrtf(warp_sum(s));
  const float d = fmaxf(n, NORM_EPS);
  for (int c = lane; c < C; c += 32) {
    const float v = xr[c] / d;
    y[static_cast<long long>(r) * C + c] = v;
    if (y_bf16) y_bf16[static_cast<long long>(r) * C + c] = __float2bfloat16_rn(v);
  }
  if (lane == 0) norm[r] = n;
}

// g = dy (+ dy2);  dx = (g - y (y . g)) / ||x|| where ||x|| >= eps, else g / eps (the clamp passes no gradient to the
// norm).  Written as bf16: it feeds the projection's dgrad / wgrad GEMMs.
__global__ void __launch_bounds__(128)
lfvila_normalize_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ dy2, const float* __restrict__ y,
                            const float* __restrict__ norm, __nv_bfloat16* __restrict__ dx, int rows, int C) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const long long o = static_cast<long long>(r) * C;
  const float n = norm[r];
  const bool clamped = !(n >= NORM_EPS);
  float s = 0.f;
  if (!clamped) {
    for (int c = lane; c < C; c += 32) {
      const float g = (dy ? dy[o + c] : 0.f) + (dy2 ? dy2[o + c] : 0.f);
      s += g * y[o + c];
    }
    s = warp_sum(s);
  }
  const float d = clamped ? NORM_EPS : n;
  for (int c = lane; c < C; c += 32) {
    const float g = (dy ? dy[o + c] : 0.f) + (dy2 ? dy2[o + c] : 0.f);
    dx[o + c] = __float2bfloat16_rn((clamped ? g : g - y[o + c] * s) / d);
  }
}

// --------------------------------------------------------------------------------- cross-entropy, accuracy
// One CTA over all B rows, one warp per row at a time.  Row r with label t: lse = max + log(sum exp(l - max)),
// loss_r = lse - l[t]; correct_r = (first index of the maximum == t).  Label -100 (CrossEntropyLoss's ignore_index) leaves
// the row out of the loss mean; any other label outside [0, n) makes the row's loss NaN (torch raises there).
// loss = sum_r loss_r / count and acc = sum_r correct_r / B, summed by one thread in row order.  pred (optional) receives
// the logits compacted to row pitch n (the classifier GEMM writes them with a padded pitch).
constexpr int CE_THREADS = 256, CE_WARPS = CE_THREADS / 32;
constexpr int CE_MAX_ROWS = 4096;
constexpr int64_t IGNORE_INDEX = -100;

// (v, i) beats (m, j) under torch's rule: a NaN beats any number, a larger value beats a smaller one, and between equals
// (or two NaNs) the lower index wins.
__device__ __forceinline__ bool beats(float v, int i, float m, int j) {
  if (isnan(v) || isnan(m)) return isnan(v) && (!isnan(m) || i < j);
  return v > m || (v == m && i < j);
}

__global__ void __launch_bounds__(CE_THREADS)
lfvila_ce_fwd_kernel(const float* __restrict__ logits, long long ld, const int64_t* __restrict__ labels, int B, int n,
                     float* __restrict__ pred, float* __restrict__ lse_out, float* __restrict__ loss, float* __restrict__ acc) {
  extern __shared__ float ce_smem[];       // row loss [B] | row correct [B] | row counted [B]
  float* s_loss = ce_smem;
  float* s_ok = ce_smem + B;
  float* s_cnt = ce_smem + 2 * B;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < B; r += CE_WARPS) {
    const float* l = logits + static_cast<long long>(r) * ld;
    float m = -INFINITY;
    int mi = 0x7fffffff;
    for (int c = lane; c < n; c += 32) {
      const float v = l[c];
      if (pred) pred[static_cast<long long>(r) * n + c] = v;
      if (beats(v, c, m, mi)) {
        m = v;
        mi = c;
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o);
      const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
      if (beats(om, oi, m, mi)) {
        m = om;
        mi = oi;
      }
    }
    float s = 0.f;
    for (int c = lane; c < n; c += 32) s += expf(l[c] - m);
    s = warp_sum(s);
    const float lse = m + logf(s);
    if (lane == 0) {
      const int64_t t = labels[r];
      const bool ignored = t == IGNORE_INDEX;
      const bool valid = t >= 0 && t < n;
      lse_out[r] = lse;
      s_loss[r] = ignored ? 0.f : valid ? lse - l[t] : NAN;
      s_cnt[r] = ignored ? 0.f : 1.f;
      s_ok[r] = (mi < n && static_cast<int64_t>(mi) == t) ? 1.f : 0.f;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float sl = 0.f, so = 0.f, sc = 0.f;
    for (int r = 0; r < B; ++r) {
      sl += s_loss[r];
      so += s_ok[r];
      sc += s_cnt[r];
    }
    loss[0] = sl / sc;
    acc[0] = so / static_cast<float>(B);
  }
}

// dlogits[r, c] = d_loss / count * (softmax(l_r)[c] - [c == t_r]) (+ d_logits[r, c]), bf16 with row pitch ld_out; the
// pad columns [n, ld_out) are written as zeros (the classifier's padded weight rows must receive no gradient).
__global__ void __launch_bounds__(CE_THREADS)
lfvila_ce_bwd_kernel(const float* __restrict__ logits, long long ld, const float* __restrict__ lse,
                     const int64_t* __restrict__ labels, const float* __restrict__ d_loss, const float* __restrict__ d_logits,
                     long long ld_d, __nv_bfloat16* __restrict__ dl, long long ld_out, int B, int n) {
  __shared__ float s_scale;
  if (threadIdx.x == 0) {
    float cnt = 0.f;
    for (int r = 0; r < B; ++r) cnt += labels[r] == IGNORE_INDEX ? 0.f : 1.f;
    s_scale = d_loss ? d_loss[0] / cnt : 0.f;
  }
  __syncthreads();
  const float k = s_scale;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < B; r += CE_WARPS) {
    const long long o = static_cast<long long>(r) * ld;
    const int64_t t = labels[r];
    const bool ignored = t == IGNORE_INDEX;
    const bool valid = t >= 0 && t < n;
    const float z = lse[r];
    for (int c = lane; c < ld_out; c += 32) {
      float g = 0.f;
      if (c < n) {
        if (d_loss && !ignored) g = valid ? k * (expf(logits[o + c] - z) - (c == t ? 1.f : 0.f)) : NAN;
        if (d_logits) g += d_logits[static_cast<long long>(r) * ld_d + c];
      }
      dl[static_cast<long long>(r) * ld_out + c] = __float2bfloat16_rn(g);
    }
  }
}

}  // namespace xp

using namespace xp;

static bool misaligned16(const char* fn, const char* name, const void* p, int& rc) {
  if (aligned(p, 16)) return false;                      // NULL passes: optional operands
  rc = fail(std::string(fn) + ": " + name + " must be 16-byte aligned");
  return true;
}

static int pool_check(const char* fn, int32_t x_dtype, int32_t B, int32_t N, int32_t Hp, int32_t Wp, int32_t C) {
  if (x_dtype != XP_DTYPE_F32 && x_dtype != XP_DTYPE_F16 && x_dtype != XP_DTYPE_BF16)
    return fail(std::string(fn) + ": x dtype must be XP_DTYPE_F32, XP_DTYPE_F16 or XP_DTYPE_BF16");
  if (Hp < 2 || Wp < 3)
    return fail(std::string(fn) + ": the (2, 3) max-pool needs Hp >= 2 and Wp >= 3 (got " + std::to_string(Hp) + " x " +
                std::to_string(Wp) + ")");
  if (B < 0 || N < 1 || C < 1) return fail(std::string(fn) + ": need B >= 0, N >= 1 and C >= 1");
  if (Hp > 4096 || Wp > 4096) return fail(std::string(fn) + ": Hp and Wp must be at most 4096");
  if (static_cast<long long>(B) * N > 0x7fffffffLL) return fail(std::string(fn) + ": B * N must fit in int32");
  if ((C + 31) / 32 > 65535) return fail(std::string(fn) + ": C must be at most 65535 * 32");
  return 0;
}

extern "C" int xp_lfvila_pool_fwd(const void* x, int32_t x_dtype, float* frame_raw, void* frame_bf16, float* global_raw,
                                  void* global_bf16, uint8_t* argmax, int32_t B, int32_t N, int32_t Hp, int32_t Wp, int32_t C,
                                  void* stream) {
  const char* fn = "xp_lfvila_pool_fwd";
  if (pool_check(fn, x_dtype, B, N, Hp, Wp, C)) return -1;
  if (!x || !frame_raw || !frame_bf16 || !global_raw || !global_bf16 || !argmax) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "x", x, rc) || misaligned16(fn, "frame_raw", frame_raw, rc) ||
      misaligned16(fn, "frame_bf16", frame_bf16, rc) || misaligned16(fn, "global_raw", global_raw, rc) ||
      misaligned16(fn, "global_bf16", global_bf16, rc) || misaligned16(fn, "argmax", argmax, rc))
    return rc;
  XP_ENTER(x);
  if (B == 0) return 0;
  const dim3 grid(static_cast<unsigned>(B), static_cast<unsigned>((C + 31) / 32));
  const dim3 block(32, POOL_FRAME_LANES);
  rc = dispatch_dtype(x_dtype, fn, [&](auto t) {
    using T = decltype(t);
    lfvila_pool_fwd_kernel<T><<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const T*>(x), frame_raw, static_cast<__nv_bfloat16*>(frame_bf16), global_raw,
        static_cast<__nv_bfloat16*>(global_bf16), argmax, N, Hp, Wp, C);
    return 0;
  });
  if (rc) return rc;
  XP_CHECK_LAUNCH("lfvila_pool_fwd_kernel");
  return 0;
}

extern "C" int xp_lfvila_pool_bwd(const float* d_frame, const float* d_global, const uint8_t* argmax, void* dx,
                                  int32_t x_dtype, int32_t B, int32_t N, int32_t Hp, int32_t Wp, int32_t C, void* stream) {
  const char* fn = "xp_lfvila_pool_bwd";
  if (pool_check(fn, x_dtype, B, N, Hp, Wp, C)) return -1;
  if (!argmax || !dx) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "d_frame", d_frame, rc) || misaligned16(fn, "d_global", d_global, rc) ||
      misaligned16(fn, "argmax", argmax, rc) || misaligned16(fn, "dx", dx, rc))
    return rc;
  XP_ENTER(dx);
  const long long total = static_cast<long long>(B) * N * Hp * Wp * C;
  if (total == 0) return 0;
  long long blocks = (total + 255) / 256;
  const long long cap = 32LL * sm_count();
  if (blocks > cap) blocks = cap;
  rc = dispatch_dtype(x_dtype, fn, [&](auto t) {
    using T = decltype(t);
    lfvila_pool_bwd_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        d_frame, d_global, argmax, static_cast<T*>(dx), total, N, Hp, Wp, C);
    return 0;
  });
  if (rc) return rc;
  XP_CHECK_LAUNCH("lfvila_pool_bwd_kernel");
  return 0;
}

static int rows_check(const char* fn, int32_t rows, int32_t C) {
  if (rows < 0 || C < 1) return fail(std::string(fn) + ": need rows >= 0 and C >= 1");
  return 0;
}

extern "C" int xp_lfvila_normalize_fwd(const float* x, float* y, void* y_bf16, float* norm, int32_t rows, int32_t C,
                                       void* stream) {
  const char* fn = "xp_lfvila_normalize_fwd";
  if (rows_check(fn, rows, C)) return -1;
  if (!x || !y || !norm) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "x", x, rc) || misaligned16(fn, "y", y, rc) || misaligned16(fn, "y_bf16", y_bf16, rc) ||
      misaligned16(fn, "norm", norm, rc))
    return rc;
  XP_ENTER(x);
  if (rows == 0) return 0;
  lfvila_normalize_fwd_kernel<<<(rows + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      x, y, static_cast<__nv_bfloat16*>(y_bf16), norm, rows, C);
  XP_CHECK_LAUNCH("lfvila_normalize_fwd_kernel");
  return 0;
}

extern "C" int xp_lfvila_normalize_bwd(const float* dy, const float* dy2, const float* y, const float* norm, void* dx_bf16,
                                       int32_t rows, int32_t C, void* stream) {
  const char* fn = "xp_lfvila_normalize_bwd";
  if (rows_check(fn, rows, C)) return -1;
  if (!y || !norm || !dx_bf16) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "dy", dy, rc) || misaligned16(fn, "dy2", dy2, rc) || misaligned16(fn, "y", y, rc) ||
      misaligned16(fn, "norm", norm, rc) || misaligned16(fn, "dx", dx_bf16, rc))
    return rc;
  XP_ENTER(y);
  if (rows == 0) return 0;
  lfvila_normalize_bwd_kernel<<<(rows + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      dy, dy2, y, norm, static_cast<__nv_bfloat16*>(dx_bf16), rows, C);
  XP_CHECK_LAUNCH("lfvila_normalize_bwd_kernel");
  return 0;
}

static int ce_check(const char* fn, int64_t ld, int32_t B, int32_t n) {
  if (B < 1 || B > CE_MAX_ROWS) return fail(std::string(fn) + ": need 1 <= B <= " + std::to_string(CE_MAX_ROWS));
  if (n < 1 || ld < n) return fail(std::string(fn) + ": need n_labels >= 1 and ld >= n_labels");
  return 0;
}

extern "C" int xp_lfvila_ce_fwd(const float* logits, int64_t ld, const int64_t* labels, int32_t B, int32_t n_labels,
                                float* pred, float* lse, float* loss, float* acc, void* stream) {
  const char* fn = "xp_lfvila_ce_fwd";
  if (ce_check(fn, ld, B, n_labels)) return -1;
  if (!logits || !labels || !lse || !loss || !acc) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "logits", logits, rc) || misaligned16(fn, "labels", labels, rc) || misaligned16(fn, "pred", pred, rc) ||
      misaligned16(fn, "lse", lse, rc))
    return rc;
  XP_ENTER(logits);
  lfvila_ce_fwd_kernel<<<1, CE_THREADS, 3 * B * sizeof(float), static_cast<cudaStream_t>(stream)>>>(
      logits, ld, labels, B, n_labels, pred, lse, loss, acc);
  XP_CHECK_LAUNCH("lfvila_ce_fwd_kernel");
  return 0;
}

extern "C" int xp_lfvila_ce_bwd(const float* logits, int64_t ld, const float* lse, const int64_t* labels, const float* d_loss,
                                const float* d_logits, int64_t ld_d, void* dlogits_bf16, int64_t ld_out, int32_t B,
                                int32_t n_labels, void* stream) {
  const char* fn = "xp_lfvila_ce_bwd";
  if (ce_check(fn, ld, B, n_labels)) return -1;
  if (ld_out < n_labels || (d_logits && ld_d < n_labels))
    return fail(std::string(fn) + ": ld_out and ld_d must be at least n_labels");
  if (!logits || !lse || !labels || !dlogits_bf16) return fail(std::string(fn) + ": null operand");
  int rc = 0;
  if (misaligned16(fn, "logits", logits, rc) || misaligned16(fn, "lse", lse, rc) || misaligned16(fn, "labels", labels, rc) ||
      misaligned16(fn, "d_logits", d_logits, rc) || misaligned16(fn, "dlogits", dlogits_bf16, rc))
    return rc;
  XP_ENTER(logits);
  lfvila_ce_bwd_kernel<<<1, CE_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      logits, ld, lse, labels, d_loss, d_logits, ld_d, static_cast<__nv_bfloat16*>(dlogits_bf16), ld_out, B, n_labels);
  XP_CHECK_LAUNCH("lfvila_ce_bwd_kernel");
  return 0;
}
