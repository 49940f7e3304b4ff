// Decoded uint8 frames of any size to the bf16 patch matrix, with the reference's whole input transform fused in:
// `.permute(0,3,1,2).float() / 255.` (dataset_pretrain_stage1_all_source.py:182), then init_transform_dict_simple
// (dataloader.py:209-233): Resize([S, S], BICUBIC) + CenterCrop(S) + Normalize(mean, std).  The pinned torchvision 0.9.0
// runs that Resize on a float tensor as F.interpolate(mode="bicubic", align_corners=False): A = -0.75, border-clamped
// taps, no antialias, no clamp of the result; CenterCrop(S) of an S x S image is the identity.
//
// Work item: one band (the p output rows of one patch row of one frame) x one tile of at most kTileCols output columns.
// A block stages the horizontal pass of every source row the band's taps touch in shared memory (each such row is read
// once per band and tile), then runs the vertical pass and writes every output element once, straight into the patch
// matrix.  When the band needs more source rows than the shared-memory budget holds (downscales by more than about
// 20 / p), it is processed in consecutive runs of output rows, which re-read only the up to three rows their windows
// share.  Items are walked with a 64-bit grid-stride loop, so the frame count is limited by memory alone.
//
// Arithmetic: the source coordinate scale * (d + 0.5) - 0.5 (scale = in / out, d + 0.5 in fp32) rounded once to fp32, a
// fused multiply-add, as torch's compiled CPU loop forms it; explicit _rn intrinsics, since the library builds with
// --use_fast_math.  The floor index and t are then torch's bit for bit.
// The four cubic weights are evaluated in float64 from that t and rounded once to fp32.  Taps are accumulated in fp32 in
// a fixed order (horizontal j = 0..3, then vertical i = 0..3), then (acc / 255 - mean) / std with IEEE operations and one
// rounding to bf16: bitwise repeatable, and at H = W = S (weights 0, 1, 0, 0) the bits of xp_vip_patchify_u8.
#include <algorithm>
#include <cmath>

#include "../../include/xpretrain_b200.h"
#include "common.h"

namespace xp {
namespace {

constexpr int kThreads = 256;
constexpr int kTileCols = 256;                 // most output columns per work item
constexpr int kSmemBudget = 64 * 1024;         // staged rows beyond the fixed tables, unless 4 rows need more
constexpr int kMaxSize = 4096;
// fixed tables (kTileCols x-taps + up to kMaxSize y-taps, 20 bytes each) + 4 staged rows of kTileCols columns
constexpr int kSmemMax = 20 * (kTileCols + kMaxSize) + 4 * 12 * kTileCols;

// upsample_bicubic2d's source index and t (align_corners=False, cubic: no clamp of a negative coordinate)
__device__ __forceinline__ void source_tap(int d, float scale, int n_in, int& i, float& t) {
  const float real = __fmaf_rn(scale, __fadd_rn(static_cast<float>(d), 0.5f), -0.5f);
  i = min(static_cast<int>(floorf(real)), n_in - 1);
  t = fminf(fmaxf(__fsub_rn(real, static_cast<float>(i)), 0.f), 1.f);
}

// the cubic convolution weights of taps i-1 .. i+2 at t, float64, rounded once to fp32
__device__ __forceinline__ float4 cubic_weights(float t) {
  const double A = -0.75, x = t;
  auto near = [&](double v) { return ((A + 2.0) * v - (A + 3.0)) * v * v + 1.0; };        // |v| <= 1
  auto far = [&](double v) { return ((A * v - 5.0 * A) * v + 8.0 * A) * v - 4.0 * A; };    // 1 < |v| < 2
  return make_float4(static_cast<float>(far(x + 1.0)), static_cast<float>(near(x)), static_cast<float>(near(1.0 - x)),
                     static_cast<float>(far(2.0 - x)));
}

__global__ void __launch_bounds__(kThreads)
resize_patchify_u8_kernel(const uint8_t* __restrict__ src, __nv_bfloat16* __restrict__ out, long long n_items, int H,
                          int W, int S, int p, int tiles, int tile_w, int rows_cap, float scale_y, float scale_x,
                          float m0, float m1, float m2, float s0, float s1, float s2) {
  extern __shared__ float4 smem4[];
  float4* xw = smem4;                                               // [tile_w]
  float4* yw = xw + tile_w;                                         // [p]
  int* xi = reinterpret_cast<int*>(yw + p);                         // [tile_w]
  int* yi = xi + tile_w;                                            // [p]
  float* hrow = reinterpret_cast<float*>(yi + p);                   // [rows_cap][3][tile_w]
  const int gs = S / p, kp = 3 * p * p, ld = (kp + 7) & ~7, tid = threadIdx.x;
  const long long row_bytes = static_cast<long long>(W) * 3;

  for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int tile = static_cast<int>(item % tiles);
    const long long band = item / tiles;                              // frame * gs + patch row
    const int ph = static_cast<int>(band % gs);
    const uint8_t* frame = src + (band / gs) * static_cast<long long>(H) * row_bytes;
    __nv_bfloat16* dst = out + band * gs * ld;                        // the band's gs patch rows, contiguous
    const int x0 = tile * tile_w, cw = min(tile_w, S - x0);
    __syncthreads();                                                  // the previous item is done with the tables
    for (int j = tid; j < cw; j += kThreads) {
      float t;
      source_tap(x0 + j, scale_x, W, xi[j], t);
      xw[j] = cubic_weights(t);
    }
    for (int k = tid; k < p; k += kThreads) {
      float t;
      source_tap(ph * p + k, scale_y, H, yi[k], t);
      yw[k] = cubic_weights(t);
    }
    if (ld != kp) {                                                   // pad columns of the patches starting in this tile
      for (int pw = (x0 + p - 1) / p; pw * p < x0 + cw; ++pw)
        for (int c = kp + tid; c < ld; c += kThreads) dst[static_cast<long long>(pw) * ld + c] = __float2bfloat16_rn(0.f);
    }
    __syncthreads();

    for (int k0 = 0; k0 < p;) {
      // the longest run of output rows k0 .. k1-1 whose source window [r_lo, r_hi] fits the staged rows (4 always do)
      const int r_lo = max(yi[k0] - 1, 0);
      int k1 = k0 + 1;
      while (k1 < p && min(yi[k1] + 2, H - 1) - r_lo < rows_cap) ++k1;
      const int rows = min(yi[k1 - 1] + 2, H - 1) - r_lo + 1;

      for (int e = tid; e < rows * cw; e += kThreads) {               // horizontal pass, one (row, column) per step
        const int r = e / cw, j = e - r * cw;
        const uint8_t* line = frame + static_cast<long long>(r_lo + r) * row_bytes;
        const float4 w = xw[j];
        const float wv[4] = {w.x, w.y, w.z, w.w};
        float acc[3];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint8_t* px = line + min(max(xi[j] - 1 + q, 0), W - 1) * 3;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const float v = static_cast<float>(px[c]);
            acc[c] = q == 0 ? __fmul_rn(wv[0], v) : __fmaf_rn(wv[q], v, acc[c]);
          }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) hrow[(r * 3 + c) * tile_w + j] = acc[c];
      }
      __syncthreads();

      const int n = (k1 - k0) * 3 * cw;
      for (int e = tid; e < n; e += kThreads) {                       // vertical pass, one output element per step
        const int rest = e / cw, j = e - rest * cw;
        const int c = rest % 3, kh = k0 + rest / 3;
        const float4 w = yw[kh];
        const float wv[4] = {w.x, w.y, w.z, w.w};
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int r = min(max(yi[kh] - 1 + q, 0), H - 1) - r_lo;
          const float h = hrow[(r * 3 + c) * tile_w + j];
          acc = q == 0 ? __fmul_rn(wv[0], h) : __fmaf_rn(wv[q], h, acc);
        }
        const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
        const float v = __fdiv_rn(__fsub_rn(__fdiv_rn(acc, 255.f), mean), sd);
        const int x = x0 + j, pw = x / p;
        dst[static_cast<long long>(pw) * ld + c * p * p + kh * p + (x - pw * p)] = __float2bfloat16_rn(v);
      }
      k0 = k1;
      __syncthreads();                                                // before the next run overwrites the staged rows
    }
  }
}

}  // namespace
}  // namespace xp

using namespace xp;

extern "C" int xp_vip_resize_patchify_u8(const uint8_t* frames_hwc, void* patches_bf16, int64_t frames, int32_t H,
                                         int32_t W, int32_t S, int32_t patch, const float* mean3, const float* std3,
                                         void* stream) {
  XP_ENTER(frames_hwc);
  if (H < 1 || W < 1 || S < 1 || H > kMaxSize || W > kMaxSize || S > kMaxSize)
    return fail("xp_vip_resize_patchify_u8: H, W and S must lie in [1, 4096]");
  if (patch < 1 || S % patch) return fail("xp_vip_resize_patchify_u8: patch must divide S");
  if (frames < 0) return fail("xp_vip_resize_patchify_u8: frames must be >= 0");
  if (!aligned(patches_bf16, 16)) return fail("xp_vip_resize_patchify_u8: patches must be 16-byte aligned");
  const int tiles = (S + kTileCols - 1) / kTileCols, tile_w = (S + tiles - 1) / tiles;
  const float scale_y = static_cast<float>(H) / static_cast<float>(S), scale_x = static_cast<float>(W) / static_cast<float>(S);
  // source rows one band touches: at most ceil((p - 1) * scale_y) + 5, and never more than H
  const long long band_rows = std::min<long long>(H, static_cast<long long>(std::ceil((patch - 1) * static_cast<double>(scale_y))) + 5);
  const int fixed = 20 * (tile_w + patch), row = 12 * tile_w;
  const int rows_cap = static_cast<int>(std::max<long long>(4, std::min<long long>(band_rows, (kSmemBudget - fixed) / row)));
  const int smem = fixed + rows_cap * row;
  if (smem > kSmemMax) return fail("xp_vip_resize_patchify_u8: shared-memory plan exceeds its limit");
  const long long items = frames * (S / patch) * tiles;
  if (items == 0) return 0;
  if (smem_limit<resize_patchify_u8_kernel>(kSmemMax) != 0) return -1;
  int per_sm = 0;
  XP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resize_patchify_u8_kernel, kThreads, smem));
  const long long grid = std::min<long long>(items, static_cast<long long>(std::max(per_sm, 1)) * sm_count());
  resize_patchify_u8_kernel<<<static_cast<unsigned>(grid), kThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      frames_hwc, static_cast<__nv_bfloat16*>(patches_bf16), items, H, W, S, patch, tiles, tile_w, rows_cap, scale_y,
      scale_x, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
  XP_CHECK_LAUNCH("resize_patchify_u8_kernel");
  return 0;
}
