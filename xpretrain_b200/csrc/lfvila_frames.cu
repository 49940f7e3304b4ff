// Decoded uint8 frames to Swin-3D's bf16 patch matrix, with LF-VILA's input transform fused in: `.float() / 255`
// (video_classification_dataset.py:84), then init_transform_dict (dataloader.py:94-121) as the pinned torchvision 0.11 runs
// it on a float tensor:
//   val / test  Resize([240, 428]) + CenterCrop([216, 385]) + Resize(input_res) + Normalize
//   train       RandomResizedCrop(input_res) (a crop of the frame, then one Resize) + RandomHorizontalFlip + Normalize
// Both are "stage A: resize the frame to Ha x Wa; crop a box; stage B: resize the box to Ho x Wo; mirror the columns if
// flip", with stage A the identity (weight exactly 1) in training.  Every resize is F.interpolate(mode="bilinear",
// align_corners=False) without antialias; stage B's taps are clamped to the box, not the frame.
//
// The composite is separable: per output row and per output column, 2 stage-B taps of 2 stage-A taps each, i.e. 4 source
// indices (not necessarily distinct or contiguous) with weights w_B * w_A.  Each coordinate is torch's fp32 value
// scale * (d + 0.5) - 0.5 (scale = in / out) rounded once, a fused multiply-add as torch's compiled CPU loop forms it,
// clamped at 0; the products w_B * w_A are formed in float64 and rounded once to fp32.
//
// Work item: one band (the 8 output rows of one patch row of one frame) x one tile of at most kTileCols output columns.
// Warp 0 gathers the band's 32 row taps into at most 32 distinct source rows; the block runs the horizontal pass of each
// of them once into shared memory, then the vertical pass, and writes every output element once, 8 columns (one patch
// row of one channel, 16 bytes) per step.  Taps accumulate in fp32 in a fixed order (horizontal q = 0..3, then vertical
// q = 0..3), then (acc / 255 - mean) / std with IEEE operations (the library builds with --use_fast_math) and one rounding
// to bf16: bitwise repeatable.  Items are walked with a 64-bit grid-stride loop over 64-bit source offsets.
#include <algorithm>

#include "../../include/xpretrain_b200.h"
#include "common.h"

namespace xp {
namespace {

constexpr int kThreads = 256;
constexpr int kP = 8;                          // Swin-3D's spatial patch
constexpr int kCols = 3 * kP * kP;             // 192 patch-matrix columns, (c, kh, kw)
constexpr int kTileCols = 256;                 // most output columns per work item
constexpr int kBandRows = 4 * kP;              // most distinct source rows of one band
constexpr int kMaxSize = 4096;

__host__ __device__ constexpr int row_pitch(int tile_w) { return tile_w + 4; }   // odd multiple of 16 bytes: no conflicts
__host__ __device__ constexpr int smem_bytes(int tile_w) {
  return 32 * tile_w + 16 * kP + 8 * kBandRows + 4 * 3 * kBandRows * row_pitch(tile_w);
}

// torch's bilinear source index, neighbour and lambda along one axis (align_corners=False; a negative coordinate is 0)
__device__ __forceinline__ void linear_tap(int d, float scale, int n_in, int& i0, int& i1, float& t) {
  const float real = fmaxf(__fmaf_rn(scale, __fadd_rn(static_cast<float>(d), 0.5f), -0.5f), 0.f);
  i0 = min(static_cast<int>(floorf(real)), n_in - 1);
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  t = fminf(fmaxf(__fsub_rn(real, static_cast<float>(i0)), 0.f), 1.f);
}

// Output index o of one axis -> 4 source indices and fp32 weights: stage B over the box [box0, box0 + len) of the stage-A
// image (n_a wide), then stage A over the n_src source pixels.  A box index is clamped to the stage-A image, so a box the
// caller failed to validate still reads inside the frame.
__device__ __forceinline__ void composite_taps(int o, float scale_b, int box0, int len, float scale_a, int n_a, int n_src,
                                               int4& idx, float4& w) {
  int b0, b1;
  float tb;
  linear_tap(o, scale_b, len, b0, b1, tb);
  int s[4];
  double ws[4];
  const int bb[2] = {b0, b1};
  const double wb[2] = {1.0 - static_cast<double>(tb), static_cast<double>(tb)};
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int a = min(max(box0 + bb[k], 0), n_a - 1);
    float ta;
    linear_tap(a, scale_a, n_src, s[2 * k], s[2 * k + 1], ta);
    ws[2 * k] = wb[k] * (1.0 - static_cast<double>(ta));
    ws[2 * k + 1] = wb[k] * static_cast<double>(ta);
  }
  idx = make_int4(s[0], s[1], s[2], s[3]);
  w = make_float4(static_cast<float>(ws[0]), static_cast<float>(ws[1]), static_cast<float>(ws[2]), static_cast<float>(ws[3]));
}

__global__ void __launch_bounds__(kThreads)
lfvila_frames_kernel(const uint8_t* __restrict__ src, const int* __restrict__ params, __nv_bfloat16* __restrict__ out,
                     long long n_items, int N, int H, int W, int Ha, int Wa, int Ho, int Wo, int tiles, int tile_w,
                     float scale_ay, float scale_ax, float m0, float m1, float m2, float s0, float s1, float s2) {
  extern __shared__ float4 smem4[];
  float4* xw = smem4;                                               // [tile_w]
  float4* yw = xw + tile_w;                                         // [kP]
  int4* xi = reinterpret_cast<int4*>(yw + kP);                      // [tile_w]
  int* slot = reinterpret_cast<int*>(xi + tile_w);                  // [kP * 4]: staged row of each row tap
  int* rows = slot + kBandRows;                                     // [kBandRows]: source row of each staged row
  float* hrow = reinterpret_cast<float*>(rows + kBandRows);         // [kBandRows][3][pitch]
  __shared__ int n_rows;
  const int gh = Ho / kP, gw = Wo / kP, pitch = row_pitch(tile_w), tid = threadIdx.x;
  const long long row_bytes = static_cast<long long>(W) * 3;

  for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int tile = static_cast<int>(item % tiles);
    const long long band = item / tiles;                              // frame * gh + patch row
    const int ph = static_cast<int>(band % gh);
    const long long frame_idx = band / gh;
    const int* pr = params + (frame_idx / N) * 5;
    const int top = pr[0], left = pr[1], bh = pr[2], bw = pr[3], flip = pr[4];
    const float scale_by = __fdiv_rn(static_cast<float>(bh), static_cast<float>(Ho));
    const float scale_bx = __fdiv_rn(static_cast<float>(bw), static_cast<float>(Wo));
    const uint8_t* frame = src + frame_idx * static_cast<long long>(H) * row_bytes;
    const int x0 = tile * tile_w, cw = min(tile_w, Wo - x0);
    __nv_bfloat16* dst = out + (band * gw + x0 / kP) * kCols;        // the tile's first patch of this band
    __syncthreads();                                                  // the previous item is done with the tables
    for (int j = tid; j < cw; j += kThreads) {
      const int x = x0 + j;
      composite_taps(flip ? Wo - 1 - x : x, scale_bx, left, bw, scale_ax, Wa, W, xi[j], xw[j]);
    }
    if (tid < 32) {                                                   // lane = kh * 4 + q: the band's row taps
      int4 idx;
      float4 w;
      composite_taps(ph * kP + tid / 4, scale_by, top, bh, scale_ay, Ha, H, idx, w);
      if (tid % 4 == 0) yw[tid / 4] = w;
      const int q = tid % 4;
      const int v = q == 0 ? idx.x : (q == 1 ? idx.y : (q == 2 ? idx.z : idx.w));
      const unsigned same = __match_any_sync(0xffffffffu, v);
      const int leader = __ffs(same) - 1;                             // the first lane holding v
      const unsigned firsts = __ballot_sync(0xffffffffu, leader == tid);
      const int s = __popc(firsts & ((1u << leader) - 1u));
      slot[tid] = s;
      if (leader == tid) rows[s] = v;
      if (tid == 0) n_rows = __popc(firsts);
    }
    __syncthreads();

    const int nr = n_rows;
    for (int e = tid; e < nr * cw; e += kThreads) {                  // horizontal pass, one (row, column) per step
      const int r = e / cw, j = e - r * cw;
      const uint8_t* line = frame + static_cast<long long>(rows[r]) * row_bytes;
      const int4 xs = xi[j];
      const float4 w = xw[j];
      const int sx[4] = {xs.x, xs.y, xs.z, xs.w};
      const float wv[4] = {w.x, w.y, w.z, w.w};
      float acc[3];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint8_t* px = line + sx[q] * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float v = static_cast<float>(px[c]);
          acc[c] = q == 0 ? __fmul_rn(wv[0], v) : __fmaf_rn(wv[q], v, acc[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) hrow[(r * 3 + c) * pitch + j] = acc[c];
    }
    __syncthreads();

    // vertical pass: one 16-byte run (8 columns kw of one (c, kh) of one patch) per step, consecutive steps consecutive runs
    const int n = (cw / kP) * 3 * kP;
    for (int e = tid; e < n; e += kThreads) {
      const int pw = e / (3 * kP), run = e - pw * 3 * kP;            // run = c * 8 + kh: the column block c*64 + kh*8
      const int c = run / kP, kh = run - c * kP;
      const float4 w = yw[kh];
      const float wv[4] = {w.x, w.y, w.z, w.w};
      const float* h[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) h[q] = hrow + (slot[kh * 4 + q] * 3 + c) * pitch + pw * kP;
      const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
      __align__(16) __nv_bfloat16 v[kP];
#pragma unroll
      for (int kw = 0; kw < kP; ++kw) {
        float acc = __fmul_rn(wv[0], h[0][kw]);
#pragma unroll
        for (int q = 1; q < 4; ++q) acc = __fmaf_rn(wv[q], h[q][kw], acc);
        v[kw] = __float2bfloat16_rn(__fdiv_rn(__fsub_rn(__fdiv_rn(acc, 255.f), mean), sd));
      }
      *reinterpret_cast<uint4*>(dst + static_cast<long long>(pw) * kCols + run * kP) = *reinterpret_cast<const uint4*>(v);
    }
  }
}

}  // namespace
}  // namespace xp

using namespace xp;

extern "C" int xp_lfvila_frames_patchify_u8(const uint8_t* frames_hwc, const int32_t* params, void* patches_bf16,
                                            int32_t clips, int32_t N, int32_t H, int32_t W, int32_t Ha, int32_t Wa,
                                            int32_t Ho, int32_t Wo, int32_t patch, const float* mean3, const float* std3,
                                            void* stream) {
  XP_ENTER(patches_bf16);
  auto in_range = [](int v) { return v >= 1 && v <= kMaxSize; };
  if (!in_range(H) || !in_range(W) || !in_range(Ha) || !in_range(Wa) || !in_range(Ho) || !in_range(Wo))
    return fail("xp_lfvila_frames_patchify_u8: H, W, Ha, Wa, Ho and Wo must lie in [1, 4096]");
  if (patch != kP) return fail("xp_lfvila_frames_patchify_u8: patch must be 8 (Swin-3D's patch)");
  if (Ho % patch || Wo % patch) return fail("xp_lfvila_frames_patchify_u8: patch must divide Ho and Wo");
  if (clips < 0 || N < 0) return fail("xp_lfvila_frames_patchify_u8: clips and N must be >= 0");
  if (!aligned(patches_bf16, 16)) return fail("xp_lfvila_frames_patchify_u8: patches must be 16-byte aligned");
  const int tiles = (Wo + kTileCols - 1) / kTileCols;
  const int tile_w = ((Wo + tiles - 1) / tiles + kP - 1) / kP * kP;
  const long long items = static_cast<long long>(clips) * N * (Ho / kP) * tiles;
  if (items == 0) return 0;
  const int smem = smem_bytes(tile_w);
  if (smem_limit<lfvila_frames_kernel>(smem_bytes(kTileCols)) != 0) return -1;
  const float scale_ay = static_cast<float>(H) / static_cast<float>(Ha), scale_ax = static_cast<float>(W) / static_cast<float>(Wa);
  int per_sm = 0;
  XP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lfvila_frames_kernel, kThreads, smem));
  const long long grid = std::min<long long>(items, static_cast<long long>(std::max(per_sm, 1)) * sm_count());
  lfvila_frames_kernel<<<static_cast<unsigned>(grid), kThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      frames_hwc, params, static_cast<__nv_bfloat16*>(patches_bf16), items, N, H, W, Ha, Wa, Ho, Wo, tiles, tile_w,
      scale_ay, scale_ax, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
  XP_CHECK_LAUNCH("lfvila_frames_kernel");
  return 0;
}
