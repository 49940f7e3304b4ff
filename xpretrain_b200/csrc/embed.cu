// Embedding-side kernels of the CLIP-ViP path (all HBM-/latency-bound, index arithmetic bit-exact):
//   * im2col of the stride-16 patch conv (CLIP_ViP.py:157-159,178-179) so the conv runs on the wgmma GEMM,
//   * the position/temporal add table and the cls / video-proxy rows (CLIP_ViP.py:170-176,183-195),
//   * their backward (scatter into class_embedding, added_cls, position_embedding, temporal_embedding),
//   * CLIP text embeddings forward/backward (CLIP_ViP.py:222-225) and EOS pooling index (CLIP_ViP.py:776).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

// F.interpolate(mode="linear", align_corners=False) source taps for output index i (CLIP_ViP.py:172-174).
__device__ __forceinline__ void linear_taps(int i, int n_in, int n_out, int& i0, int& i1, float& w1) {
  if (n_in == n_out) {
    i0 = i1 = i;
    w1 = 0.f;
    return;
  }
  float src = (static_cast<float>(i) + 0.5f) * (static_cast<float>(n_in) / static_cast<float>(n_out)) - 0.5f;
  if (src < 0.f) src = 0.f;
  i0 = static_cast<int>(src);
  if (i0 > n_in - 1) i0 = n_in - 1;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  w1 = src - static_cast<float>(i0);
}

// ------------------------------------------------------------------------ im2col
// video [F, 3, H, W] (F = B*T frames) -> patches [F * (H/p) * (W/p), 3*p*p] bf16, column = c*p*p + kh*p + kw
// (the flattening order of Conv2d.weight [out, c, kh, kw]); patch order row-major over the grid (flatten(2), :179).
template <typename T>
__global__ void __launch_bounds__(256)
patchify_kernel(const T* __restrict__ video, __nv_bfloat16* __restrict__ out, long long frames, int H, int W, int p) {
  // one thread per 8 consecutive pixels of an image row; p % 8 == 0
  const int wchunks = W / 8;
  const long long total = frames * 3 * H * wchunks;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int wc = static_cast<int>(idx % wchunks);
  long long rest = idx / wchunks;
  const int y = static_cast<int>(rest % H);
  rest /= H;
  const int c = static_cast<int>(rest % 3);
  const long long f = rest / 3;
  float v[8];
  load8(video + ((f * 3 + c) * H + y) * W + wc * 8, v);
  const int gw = W / p, gh = H / p;
  const int pw = (wc * 8) / p, kw = (wc * 8) % p, ph = y / p, kh = y % p;
  const long long row = (f * gh + ph) * gw + pw;
  store8(out + row * (3 * p * p) + c * p * p + kh * p + kw, v);
}

// uint8 frames as the decoder delivers them, [frames, H, W, 3] (HWC), to the same bf16 patch matrix, with the reference's
// input transform applied on the fly: `img_array.permute(0, 3, 1, 2).float() / 255.` (dataset_pretrain_stage1_all_source.py:182)
// followed by torchvision Normalize(mean, std) of init_transform_dict_simple (dataloader.py:209-233) for frames that already
// have the input resolution (Resize / CenterCrop to the same size are the identity).  IEEE division / subtraction in fp32
// (explicit _rn intrinsics: the library is built with --use_fast_math), then ONE rounding to bf16 — bit-identical to
// casting the reference's fp32 tensor.  A step then uploads 1 byte per sample value instead of 4.
__global__ void __launch_bounds__(256)
patchify_u8_kernel(const uint8_t* __restrict__ frames, __nv_bfloat16* __restrict__ out, long long n_frames, int H, int W, int p,
                   float m0, float m1, float m2, float s0, float s1, float s2) {
  // one thread per 8 consecutive pixels of an image row (24 contiguous bytes); p % 8 == 0, W % 8 == 0
  const int wchunks = W / 8;
  const long long total = n_frames * H * wchunks;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int wc = static_cast<int>(idx % wchunks);
  long long rest = idx / wchunks;
  const int y = static_cast<int>(rest % H);
  const long long f = rest / H;
  const uint2* src = reinterpret_cast<const uint2*>(frames + ((f * H + y) * W + wc * 8) * 3);
  const uint2 a = src[0], b = src[1], c = src[2];
  const uint32_t w[6] = {a.x, a.y, b.x, b.y, c.x, c.y};
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  const int gw = W / p, gh = H / p;
  const int pw = (wc * 8) / p, kw = (wc * 8) % p, ph = y / p, kh = y % p;
  const long long row = (f * gh + ph) * gw + pw;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float v[8];
#pragma unroll
    for (int px = 0; px < 8; ++px) {
      const int byte = px * 3 + ch;
      const float x = static_cast<float>((w[byte >> 2] >> ((byte & 3) * 8)) & 0xffu);
      v[px] = __fdiv_rn(__fsub_rn(__fdiv_rn(x, 255.f), mean[ch]), sd[ch]);
    }
    store8(out + row * (3 * p * p) + ch * p * p + kh * p + kw, v);
  }
}

// Any patch size dividing H and W (ViT-L/14: p = 14).  The patch matrix row pitch is ld = round_up(3 p^2, 8) (16-byte rows
// for TMA and the GEMM); columns [3 p^2, ld) are written as zero.  One thread per 8 consecutive columns of a patch row: a
// gather of 8 input values (the same conversion and rounding as the vectorised kernels above) and one 16-byte store.
template <typename T, bool U8>
__global__ void __launch_bounds__(256)
patchify_any_kernel(const T* __restrict__ src, __nv_bfloat16* __restrict__ out, long long frames, int H, int W, int p,
                    float m0, float m1, float m2, float s0, float s1, float s2) {
  const int kp = 3 * p * p, ld = (kp + 7) & ~7, cchunks = ld / 8;
  const int gw = W / p, gh = H / p;
  const long long total = frames * gh * gw * cchunks;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cc = static_cast<int>(idx % cchunks);
  const long long row = idx / cchunks;
  const int pw = static_cast<int>(row % gw), ph = static_cast<int>((row / gw) % gh);
  const long long f = row / (static_cast<long long>(gw) * gh);
  const float mean[3] = {m0, m1, m2}, sd[3] = {s0, s1, s2};
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = cc * 8 + i;
    v[i] = 0.f;
    if (col < kp) {
      const int c = col / (p * p), kh = (col / p) % p, kw = col % p;
      const int y = ph * p + kh, x = pw * p + kw;
      if (U8) {
        const float u = static_cast<float>(reinterpret_cast<const uint8_t*>(src)[((f * H + y) * W + x) * 3 + c]);
        v[i] = __fdiv_rn(__fsub_rn(__fdiv_rn(u, 255.f), mean[c]), sd[c]);
      } else {
        v[i] = to_f32<T>(src[((f * 3 + c) * H + y) * W + x]);
      }
    }
  }
  store8(out + row * ld + cc * 8, v);
}

// ------------------------------------------------------------ embedding tables
// table[t*L + l, :] = interp(temporal)[t, :] + pos[1 + l, :]      (bf16; the patch GEMM adds it as a periodic residual)
// x[b, m, :]       = (m == 0 ? class_embedding : added_cls[m-1]) + pos[0, :]   for m < M
__global__ void __launch_bounds__(128)
vip_embed_tables_kernel(const float* __restrict__ pos, const float* __restrict__ temporal, const float* __restrict__ cls,
                        const float* __restrict__ added, __nv_bfloat16* __restrict__ table,
                        __nv_bfloat16* __restrict__ x, int B, int T, int L, int M, int C, int Tsz, long long S) {
  const int rows_table = T * L;
  const int r = blockIdx.x;
  if (r < rows_table) {
    const int t = r / L, l = r % L;
    int i0, i1;
    float w1;
    linear_taps(t, Tsz, T, i0, i1, w1);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      float tv = 0.f;
      if (temporal) {
        const float a = temporal[static_cast<long long>(i0) * C + c], b = temporal[static_cast<long long>(i1) * C + c];
        tv = (T == Tsz) ? a : (1.f - w1) * a + w1 * b;
      }
      table[static_cast<long long>(r) * C + c] = __float2bfloat16(tv + pos[static_cast<long long>(1 + l) * C + c]);
    }
  } else {
    const int g = r - rows_table;  // 0 .. B*M-1
    const int b = g / M, m = g % M;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const float e = (m == 0) ? cls[c] : added[static_cast<long long>(m - 1) * C + c];
      x[(static_cast<long long>(b) * S + m) * C + c] = __float2bfloat16(e + pos[c]);
    }
  }
}

// Gradient of the embedding sum w.r.t. its parameters, accumulated in fp32.  d_patch [B, T*L, C] and
// d_global [B, M, C] are the compact halves of d_emb (patch rows / global-token rows).
__global__ void __launch_bounds__(128)
vip_embed_bwd_kernel(const __nv_bfloat16* __restrict__ d_patch, const __nv_bfloat16* __restrict__ d_global,
                     float* __restrict__ d_pos, float* __restrict__ d_temporal, float* __restrict__ d_cls,
                     float* __restrict__ d_added, int B, int T, int L, int M, int C, int Tsz) {
  const int j = blockIdx.x;  // sequence position 0..M+T*L-1
  const int c0 = threadIdx.x * 8;
  if (c0 >= C) return;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const __nv_bfloat16* src = j < M ? d_global + static_cast<long long>(j) * C : d_patch + static_cast<long long>(j - M) * C;
  const long long bstride = j < M ? static_cast<long long>(M) * C : static_cast<long long>(T) * L * C;
#pragma unroll 4
  for (int b = 0; b < B; ++b) {
    float v[8];
    load8(src + b * bstride + c0, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += v[i];
  }
  if (j < M) {
    // d_cls / d_added are optional like d_temporal: a caller without that gradient passes NULL
    float* dst = (j == 0) ? d_cls : (d_added != nullptr ? d_added + static_cast<long long>(j - 1) * C : nullptr);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (dst != nullptr) atomicAdd(dst + c0 + i, acc[i]);
      atomicAdd(d_pos + c0 + i, acc[i]);
    }
  } else {
    const int t = (j - M) / L, l = (j - M) % L;
#pragma unroll
    for (int i = 0; i < 8; ++i) atomicAdd(d_pos + static_cast<long long>(1 + l) * C + c0 + i, acc[i]);
    if (d_temporal) {
      int i0, i1;
      float w1;
      linear_taps(t, Tsz, T, i0, i1, w1);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (T == Tsz) {
          atomicAdd(d_temporal + static_cast<long long>(i0) * C + c0 + i, acc[i]);
        } else {
          atomicAdd(d_temporal + static_cast<long long>(i0) * C + c0 + i, (1.f - w1) * acc[i]);
          atomicAdd(d_temporal + static_cast<long long>(i1) * C + c0 + i, w1 * acc[i]);
        }
      }
    }
  }
}

// -------------------------------------------------------------- text embeddings
__global__ void __launch_bounds__(128)
text_embed_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                      __nv_bfloat16* __restrict__ x, int Lt, int C, int vocab, int* __restrict__ err) {
  const long long r = blockIdx.x;  // b*Lt + s
  const int s = static_cast<int>(r % Lt);
  long long id = ids[r];
  if (id < 0 || id >= vocab) {  // nn.Embedding raises on out-of-range ids; flag it for the host
    if (threadIdx.x == 0) atomicExch(err, 1);
    id = 0;
  }
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4) {
    const float4 a = *reinterpret_cast<const float4*>(tok + id * C + c);
    const float4 b = *reinterpret_cast<const float4*>(pos + static_cast<long long>(s) * C + c);
    uint2 o;
    o.x = pack_bf16(a.x + b.x, a.y + b.y);
    o.y = pack_bf16(a.z + b.z, a.w + b.w);
    *reinterpret_cast<uint2*>(x + r * C + c) = o;
  }
}
__global__ void __launch_bounds__(128)
text_embed_bwd_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ dx, float* __restrict__ d_tok,
                      float* __restrict__ d_pos, int Lt, int C, int vocab) {
  const long long r = blockIdx.x;
  const int s = static_cast<int>(r % Lt);
  long long id = ids[r];
  if (id < 0 || id >= vocab) return;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float g = __bfloat162float(dx[r * C + c]);
    if (d_tok) atomicAdd(d_tok + id * C + c, g);
    if (d_pos) atomicAdd(d_pos + static_cast<long long>(s) * C + c, g);
  }
}

// offsets[b] = (b*Lt + argmax_s ids[b, s]) * C with the FIRST maximum (torch.argmax semantics, CLIP_ViP.py:776).
__global__ void __launch_bounds__(32)
eos_offsets_kernel(const long long* __restrict__ ids, long long* __restrict__ offsets, int* __restrict__ index, int Lt,
                   int C) {
  const int b = blockIdx.x, lane = threadIdx.x;
  long long best = LLONG_MIN;
  int best_i = 0x7fffffff;
  for (int s = lane; s < Lt; s += 32) {
    const long long v = ids[static_cast<long long>(b) * Lt + s];
    if (v > best) {
      best = v;
      best_i = s;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ov > best || (ov == best && oi < best_i)) {
      best = ov;
      best_i = oi;
    }
  }
  if (lane == 0) {
    offsets[b] = (static_cast<long long>(b) * Lt + best_i) * C;
    if (index) index[b] = best_i;
  }
}

}  // namespace xp

using namespace xp;

extern "C" int xp_vip_patchify(const void* video, int32_t dtype, void* patches_bf16, int64_t frames, int32_t H,
                               int32_t W, int32_t patch, void* stream) {
  XP_ENTER(video);
  if (patch < 1 || W % patch || H % patch) return fail("xp_vip_patchify: patch must divide H and W");
  // every path stores the patch matrix in 16-byte vectors; the p % 8 == 0 path also loads the video in 16-byte vectors
  if (!aligned(patches_bf16, 16)) return fail("xp_vip_patchify: patches must be 16-byte aligned");
  if (patch % 8 == 0 && !aligned(video, 16)) return fail("xp_vip_patchify: video must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  __nv_bfloat16* out = static_cast<__nv_bfloat16*>(patches_bf16);
  if (patch % 8) {
    const long long total = frames * (H / patch) * (W / patch) * (((3 * patch * patch + 7) & ~7) / 8);
    if (total <= 0) return 0;
    const unsigned grid = static_cast<unsigned>((total + 255) / 256);
    return dispatch_dtype(dtype, "xp_vip_patchify: dtype must be XP_DTYPE_F32 / BF16 / F16", [&](auto t) {
      using T = decltype(t);
      patchify_any_kernel<T, false><<<grid, 256, 0, st>>>(static_cast<const T*>(video), out, frames, H, W, patch, 0.f, 0.f,
                                                          0.f, 1.f, 1.f, 1.f);
      XP_CHECK_LAUNCH("patchify_any_kernel");
      return 0;
    });
  }
  const long long total = frames * 3 * H * (W / 8);
  if (total <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  return dispatch_dtype(dtype, "xp_vip_patchify: dtype must be XP_DTYPE_F32 / BF16 / F16", [&](auto t) {
    using T = decltype(t);
    patchify_kernel<T><<<grid, 256, 0, st>>>(static_cast<const T*>(video), out, frames, H, W, patch);
    XP_CHECK_LAUNCH("patchify_kernel");
    return 0;
  });
}

extern "C" int xp_vip_patchify_u8(const uint8_t* frames_hwc, void* patches_bf16, int64_t frames, int32_t H, int32_t W,
                                  int32_t patch, const float* mean3, const float* std3, void* stream) {
  XP_ENTER(frames_hwc);
  if (patch < 1 || W % patch || H % patch) return fail("xp_vip_patchify_u8: patch must divide H and W");
  if (!aligned(patches_bf16, 16)) return fail("xp_vip_patchify_u8: patches must be 16-byte aligned");
  if (patch % 8) {
    const long long total = frames * (H / patch) * (W / patch) * (((3 * patch * patch + 7) & ~7) / 8);
    if (total <= 0) return 0;
    patchify_any_kernel<uint8_t, true><<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        frames_hwc, static_cast<__nv_bfloat16*>(patches_bf16), frames, H, W, patch, mean3[0], mean3[1], mean3[2], std3[0],
        std3[1], std3[2]);
    XP_CHECK_LAUNCH("patchify_any_kernel");
    return 0;
  }
  if (!aligned(frames_hwc, 8)) return fail("xp_vip_patchify_u8: frames must be 8-byte aligned");
  const long long total = frames * H * (W / 8);
  if (total <= 0) return 0;
  patchify_u8_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      frames_hwc, static_cast<__nv_bfloat16*>(patches_bf16), frames, H, W, patch, mean3[0], mean3[1], mean3[2], std3[0], std3[1],
      std3[2]);
  XP_CHECK_LAUNCH("patchify_u8_kernel");
  return 0;
}

extern "C" int xp_vip_embed_tables(const float* pos, const float* temporal, const float* cls, const float* added,
                                   void* table_bf16, void* x_bf16, int32_t B, int32_t T, int32_t L, int32_t M,
                                   int32_t C, int32_t temporal_size, void* stream) {
  XP_ENTER(pos);
  const long long S = static_cast<long long>(M) + static_cast<long long>(T) * L;
  const int grid = T * L + B * M;
  vip_embed_tables_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      pos, temporal, cls, added, static_cast<__nv_bfloat16*>(table_bf16), static_cast<__nv_bfloat16*>(x_bf16), B, T, L,
      M, C, temporal_size, S);
  XP_CHECK_LAUNCH("vip_embed_tables_kernel");
  return 0;
}

extern "C" int xp_vip_embed_bwd(const void* d_patch_bf16, const void* d_global_bf16, float* d_pos, float* d_temporal,
                                float* d_cls, float* d_added, int32_t B, int32_t T, int32_t L, int32_t M, int32_t C,
                                int32_t temporal_size, void* stream) {
  XP_ENTER(d_patch_bf16);
  if (C % 8 || C > 1024) return fail("xp_vip_embed_bwd: C must be a multiple of 8 and <= 1024");
  if (d_pos == nullptr) return fail("xp_vip_embed_bwd: d_pos is required");
  if (!aligned(d_patch_bf16, 16) || !aligned(d_global_bf16, 16))
    return fail("xp_vip_embed_bwd: d_patch and d_global must be 16-byte aligned");
  const long long S = static_cast<long long>(M) + static_cast<long long>(T) * L;
  vip_embed_bwd_kernel<<<static_cast<unsigned>(S), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(d_patch_bf16), static_cast<const __nv_bfloat16*>(d_global_bf16), d_pos,
      d_temporal, d_cls, d_added, B, T, L, M, C, temporal_size);
  XP_CHECK_LAUNCH("vip_embed_bwd_kernel");
  return 0;
}

extern "C" int xp_text_embed_fwd(const int64_t* ids, const float* tok, const float* pos, void* x_bf16, int32_t rows,
                                 int32_t Lt, int32_t C, int32_t vocab, int32_t* err_flag, void* stream) {
  XP_ENTER(ids);
  if (C % 4) return fail("xp_text_embed_fwd: C must be a multiple of 4");
  if (!aligned(tok, 16) || !aligned(pos, 16)) return fail("xp_text_embed_fwd: tok and pos must be 16-byte aligned");
  if (!aligned(x_bf16, 8)) return fail("xp_text_embed_fwd: x must be 8-byte aligned");
  if (rows <= 0) return 0;
  text_embed_fwd_kernel<<<rows, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), tok, pos, static_cast<__nv_bfloat16*>(x_bf16), Lt, C, vocab, err_flag);
  XP_CHECK_LAUNCH("text_embed_fwd_kernel");
  return 0;
}

extern "C" int xp_text_embed_bwd(const int64_t* ids, const void* dx_bf16, float* d_tok, float* d_pos, int32_t rows,
                                 int32_t Lt, int32_t C, int32_t vocab, void* stream) {
  XP_ENTER(ids);
  if (rows <= 0) return 0;
  text_embed_bwd_kernel<<<rows, 128, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), static_cast<const __nv_bfloat16*>(dx_bf16), d_tok, d_pos, Lt, C, vocab);
  XP_CHECK_LAUNCH("text_embed_bwd_kernel");
  return 0;
}

extern "C" int xp_eos_offsets(const int64_t* ids, int64_t* offsets, int32_t* index, int32_t B, int32_t Lt, int32_t C,
                              void* stream) {
  XP_ENTER(ids);
  if (B <= 0) return 0;
  eos_offsets_kernel<<<B, 32, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const long long*>(ids),
                                                                     reinterpret_cast<long long*>(offsets), index, Lt, C);
  XP_CHECK_LAUNCH("eos_offsets_kernel");
  return 0;
}
