// Video-proxy (ViP) attention of CLIP-ViP, forward and backward, one CTA per (batch, head, frame), for frames of
// M + L <= 208 rows (ViT-B/16 and B/32); longer frames run the streamed kernels of vip_attention_long.cu.
//
// Reference: CLIPAttention.forward2, CLIP_ViP.py:332-381.  Patch queries of frame t attend to
// [M global keys ; L keys of frame t] (:352-363); the M global queries (cls + video proxies) attend to
// all M + T*L keys (:366-375).  The reference materialises the per-frame K/V with repeat+cat; here a CTA
// stages the L frame rows and the M global rows of the fused qkv buffer once in shared memory and treats
// the global queries as extra query rows: their softmax over all frames is assembled from per-frame
// partials (max, sum, unnormalised output) by a small combine kernel.  q arrives pre-scaled by
// head_dim**-0.5 from the QKV GEMM epilogue (CLIP_ViP.py:341).
//
// Hopper path: one thread stages the operands by TMA (two boxes per matrix: the L frame rows into shared-memory rows
// [0, L), the M global rows into rows [248, 248 + M), both 1024-byte aligned for the 128B swizzle; the rows between
// are zero), completion on an mbarrier.  Two warpgroups each own 64-row tiles and run the per-block steps of
// attn_wgmma.cuh over the four staged tiles: forward fwd_step; backward pass A (key-stationary) kv_step, pass B
// (query-stationary) q_step.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "attn_wgmma.cuh"
#include "vip_attention.h"

namespace xp {

constexpr int SROWS = 256;                 // shared-memory rows per staged matrix (4 tiles of 64)
constexpr int GROW = 248;                  // first shared-memory row of the global tokens (1024-byte aligned)
constexpr int MAT_BYTES = SROWS * 128;     // one [256][64] bf16 matrix, 128B-swizzled
constexpr int TILE_BYTES = 64 * 128;       // 64 rows
constexpr int ATT_THREADS = 256;           // two warpgroups

// shared-memory row r: a frame token (r < L), a global token (GROW <= r < GROW + M) or zero padding
__device__ __forceinline__ bool row_valid(int r, const AttnDims& d) { return r < d.L || (r >= GROW && r < GROW + d.M); }
__device__ __forceinline__ bool row_global(int r) { return r >= GROW; }
__device__ __forceinline__ int row_seq(int r, const AttnDims& d) { return r >= GROW ? r - GROW : d.M + r; }
// a 64-row tile holds at least one token (tile 3 always holds the global rows)
__device__ __forceinline__ bool tile_live(int k, const AttnDims& d) { return k == 3 || 64 * k < d.L; }

// Zero the padding rows of NMAT matrices, then TMA the frame rows and global rows of each; every thread waits.
template <int NMAT>
__device__ __forceinline__ void stage_rows(uint8_t* sm, uint64_t* bar, const CUtensorMap* const (&mapL)[NMAT],
                                           const CUtensorMap* const (&mapM)[NMAT], const int (&col)[NMAT], const AttnDims& d,
                                           int b, int t) {
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
  }
  const uint32_t base = smem_u32(sm);
  for (int idx = threadIdx.x; idx < NMAT * SROWS * 8; idx += ATT_THREADS) {
    const int m = idx / (SROWS * 8), row = (idx >> 3) % SROWS;
    if (!row_valid(row, d)) st_shared_zero16(base + m * MAT_BYTES + row * 128 + (idx & 7) * 16);
  }
  fence_proxy_async_smem();     // the zero rows are read by wgmma (async proxy)
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(bar, NMAT * (d.L + d.M) * 128);
#pragma unroll
    for (int m = 0; m < NMAT; ++m) {
      tma_load_2d(sm + m * MAT_BYTES, mapL[m], bar, col[m], static_cast<int>(b * d.S + d.M + static_cast<long long>(t) * d.L));
      tma_load_2d(sm + m * MAT_BYTES + GROW * 128, mapM[m], bar, col[m], static_cast<int>(b * d.S));
    }
  }
  mbar_wait_nocall(bar, 0);
}

// ======================================================================== forward
// grid (T, H, B).  out: [B*S, C] bf16 (frame rows); lse: [B, H, S] fp32 (frame rows);
// part: [B, H, T, M, 66] fp32 = {max, sum, unnormalised out[64]} of the global queries over this frame's keys.
__global__ void __launch_bounds__(ATT_THREADS, 2)
vip_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmL, const __grid_constant__ CUtensorMap tmM,
                    __nv_bfloat16* __restrict__ out, float* __restrict__ lse, float* __restrict__ part, const AttnDims d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + 3 * MAT_BYTES);
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  {
    const CUtensorMap* const mL[3] = {&tmL, &tmL, &tmL};
    const CUtensorMap* const mM[3] = {&tmM, &tmM, &tmM};
    const int col[3] = {h * HD, d.C + h * HD, 2 * d.C + h * HD};
    stage_rows<3>(sm, bar, mL, mM, col, d, b, t);
  }
  const uint32_t sQ = smem_u32(sm), sK = sQ + MAT_BYTES, sV = sK + MAT_BYTES;
  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool mask_gg = (t != 0);   // (global query, global key) pairs belong to frame 0 only

  for (int qt = wg; qt < 4; qt += 2) {
    if (!tile_live(qt, d)) continue;
    const int r_lo = qt * 64 + wq * 16 + (lane >> 2);
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
#pragma unroll 1
    for (int kb = 0; kb < 4; ++kb) {
      if (!tile_live(kb, d)) continue;
      // masks: padding keys; for global QUERY rows, the global keys count only once (frame 0)
      fwd_step(sQ + qt * TILE_BYTES, sK + kb * TILE_BYTES, sV + kb * TILE_BYTES, o, m_run, l_run, [&](int q, int key) {
        const int k = kb * 64 + key;
        return row_valid(k, d) && !(mask_gg && row_global(qt * 64 + q) && row_global(k));
      });
    }
    quad_sum(l_run);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = r_lo + r * 8;
      if (!row_valid(row, d)) continue;
      if (row_global(row)) {   // global-query row: this frame's partial (fp32, unnormalised)
        float* p = part + (((static_cast<long long>(b) * d.H + h) * d.T + t) * d.M + (row - GROW)) * 66;
        if ((lane & 3) == 0) {
          p[0] = m_run[r];
          p[1] = l_run[r];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          p[2 + i * 8 + (lane & 3) * 2] = o[4 * i + 2 * r];
          p[2 + i * 8 + (lane & 3) * 2 + 1] = o[4 * i + 2 * r + 1];
        }
      } else {                 // frame row: normalised output + LSE
        const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
        const long long tr = token_row(d, b, t, row_seq(row, d));
        __nv_bfloat16* dst = out + tr * d.ld_o + h * HD + (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<uint32_t*>(dst + i * 8) = pack_bf16(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
        if ((lane & 3) == 0)
          lse[(static_cast<long long>(b) * d.H + h) * d.S + (tr - static_cast<long long>(b) * d.S)] = m_run[r] + logf(l_run[r]);
      }
    }
  }
}

// Merge the per-frame partials of the M global queries: grid (H, B), block 64 threads (one per head-dim column).
__global__ void __launch_bounds__(64)
vip_attn_fwd_combine_kernel(const float* __restrict__ part, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                            const AttnDims d) {
  const int h = blockIdx.x, b = blockIdx.y, c = threadIdx.x;
  for (int m = 0; m < d.M; ++m) {
    const float* p0 = part + ((static_cast<long long>(b) * d.H + h) * d.T * d.M + m) * 66;
    float mx = -INFINITY;
    for (int t = 0; t < d.T; ++t) mx = fmaxf(mx, p0[static_cast<long long>(t) * d.M * 66]);
    float l = 0.f, acc = 0.f;
    for (int t = 0; t < d.T; ++t) {
      const float* p = p0 + static_cast<long long>(t) * d.M * 66;
      const float w = __expf(p[0] - mx);
      l += p[1] * w;
      acc += p[2 + c] * w;
    }
    out[(static_cast<long long>(b) * d.S + m) * d.ld_o + h * HD + c] = __float2bfloat16(acc / l);
    if (c == 0) lse[(static_cast<long long>(b) * d.H + h) * d.S + m] = mx + logf(l);
  }
}


// ======================================================================= backward
// dqkv: [B*S, 3C] bf16 (frame rows written here; the M global rows by the combine kernel);
// gpart: [B, H, T, M, 3, 64] fp32 partial dq/dk/dv of the global rows from this frame.
__global__ void __launch_bounds__(ATT_THREADS, 1)
vip_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmL, const __grid_constant__ CUtensorMap tmM,
                    const __grid_constant__ CUtensorMap tdL, const __grid_constant__ CUtensorMap tdM,
                    const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout, const float* __restrict__ lse,
                    __nv_bfloat16* __restrict__ dqkv, float* __restrict__ gpart, const AttnDims d, float q_scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  float* s_lse = reinterpret_cast<float*>(sm + 4 * MAT_BYTES);   // lse * log2(e), +inf on padding rows
  float* s_delta = s_lse + SROWS;                                  // rowsum(dO * O)
  uint64_t* bar = reinterpret_cast<uint64_t*>(s_delta + SROWS);
  const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  {
    const CUtensorMap* const mL[4] = {&tmL, &tmL, &tmL, &tdL};
    const CUtensorMap* const mM[4] = {&tmM, &tmM, &tmM, &tdM};
    const int col[4] = {h * HD, d.C + h * HD, 2 * d.C + h * HD, h * HD};
    stage_rows<4>(sm, bar, mL, mM, col, d, b, t);
  }
  // delta_i = sum_d dO[i,d] * O[i,d] and the saved LSE per shared-memory row (8 lanes per row, 16 bytes each)
  for (int base = 0; base < SROWS; base += ATT_THREADS / 8) {
    const int row = base + (threadIdx.x >> 3), chunk = threadIdx.x & 7;
    float dot = 0.f;
    const bool valid = row_valid(row, d);
    long long tr = 0;
    if (valid) {
      tr = token_row(d, b, t, row_seq(row, d));
      const long long off = tr * d.ld_o + h * HD + chunk * 8;
      const uint4 g = *reinterpret_cast<const uint4*>(dout + off);
      const uint4 o = *reinterpret_cast<const uint4*>(out + off);
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) dot += bf16_lo(gw[i]) * bf16_lo(ow[i]) + bf16_hi(gw[i]) * bf16_hi(ow[i]);
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    dot += __shfl_xor_sync(0xffffffffu, dot, 4);
    if (chunk == 0) {
      s_delta[row] = dot;
      s_lse[row] = valid ? lse[(static_cast<long long>(b) * d.H + h) * d.S + (tr - static_cast<long long>(b) * d.S)] * LOG2E
                         : INFINITY;
    }
  }
  __syncthreads();

  const uint32_t sQ = smem_u32(sm), sK = sQ + MAT_BYTES, sV = sK + MAT_BYTES, sdO = sV + MAT_BYTES;
  const int wg = threadIdx.x >> 7, wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool mask_gg = (t != 0);
  // (query row, key row) pairs of the staged rows that enter the softmax
  const auto pair_live = [&](int q, int key) {
    return row_valid(q, d) && row_valid(key, d) && !(mask_gg && row_global(q) && row_global(key));
  };
  float* gp = gpart + ((static_cast<long long>(b) * d.H + h) * d.T + t) * d.M * 3 * HD;

  // ------------------------------------------------ pass A: key-stationary -> dK, dV
  for (int kt = wg; kt < 4; kt += 2) {
    if (!tile_live(kt, d)) continue;
    const int k_lo = kt * 64 + wq * 16 + (lane >> 2);
    float dk[32], dv[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
#pragma unroll 1
    for (int qb = 0; qb < 4; ++qb) {
      if (!tile_live(qb, d)) continue;
      kv_step(sK + kt * TILE_BYTES, sV + kt * TILE_BYTES, sQ + qb * TILE_BYTES, sdO + qb * TILE_BYTES, s_lse + qb * 64,
              s_delta + qb * 64, dk, dv, [&](int q, int key) { return pair_live(qb * 64 + q, kt * 64 + key); });
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int key = k_lo + r * 8;
      if (!row_valid(key, d)) continue;
      if (!row_global(key)) {
        __nv_bfloat16* row = dqkv + token_row(d, b, t, row_seq(key, d)) * d.ld_qkv + h * HD + (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          *reinterpret_cast<uint32_t*>(row + d.C + i * 8) = pack_bf16(dk[4 * i + 2 * r], dk[4 * i + 2 * r + 1]);
          *reinterpret_cast<uint32_t*>(row + 2 * d.C + i * 8) = pack_bf16(dv[4 * i + 2 * r], dv[4 * i + 2 * r + 1]);
        }
      } else {
        float* g = gp + static_cast<long long>(key - GROW) * 3 * HD + (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          g[HD + i * 8] = dk[4 * i + 2 * r]; g[HD + i * 8 + 1] = dk[4 * i + 2 * r + 1];
          g[2 * HD + i * 8] = dv[4 * i + 2 * r]; g[2 * HD + i * 8 + 1] = dv[4 * i + 2 * r + 1];
        }
      }
    }
  }

  // ---------------------------------------------------- pass B: query-stationary -> dQ
  for (int qt = wg; qt < 4; qt += 2) {
    if (!tile_live(qt, d)) continue;
    const int q_lo = qt * 64 + wq * 16 + (lane >> 2);
    const float lse_r[2] = {s_lse[q_lo], s_lse[q_lo + 8]}, del_r[2] = {s_delta[q_lo], s_delta[q_lo + 8]};
    float dq[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dq[i] = 0.f;
#pragma unroll 1
    for (int kb = 0; kb < 4; ++kb) {
      if (!tile_live(kb, d)) continue;
      q_step(sQ + qt * TILE_BYTES, sdO + qt * TILE_BYTES, sK + kb * TILE_BYTES, sV + kb * TILE_BYTES, lse_r, del_r, dq,
             [&](int q, int key) { return pair_live(qt * 64 + q, kb * 64 + key); });
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = q_lo + r * 8;
      if (!row_valid(q, d)) continue;
      if (!row_global(q)) {
        __nv_bfloat16* row = dqkv + token_row(d, b, t, row_seq(q, d)) * d.ld_qkv + h * HD + (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<uint32_t*>(row + i * 8) = pack_bf16(dq[4 * i + 2 * r] * q_scale, dq[4 * i + 2 * r + 1] * q_scale);
      } else {
        float* g = gp + static_cast<long long>(q - GROW) * 3 * HD + (lane & 3) * 2;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          g[i * 8] = dq[4 * i + 2 * r];
          g[i * 8 + 1] = dq[4 * i + 2 * r + 1];
        }
      }
    }
  }
}

// Sum the per-frame partial gradients of the M global rows: grid (H, B), block 192 = 3 x 64.
__global__ void __launch_bounds__(192)
vip_attn_bwd_combine_kernel(const float* __restrict__ gpart, __nv_bfloat16* __restrict__ dqkv, const AttnDims d,
                            float q_scale) {
  const int h = blockIdx.x, b = blockIdx.y;
  const int which = threadIdx.x / HD, c = threadIdx.x % HD;
  for (int m = 0; m < d.M; ++m) {
    float acc = 0.f;
    for (int t = 0; t < d.T; ++t)
      acc += gpart[((((static_cast<long long>(b) * d.H + h) * d.T + t) * d.M + m) * 3 + which) * HD + c];
    if (which == 0) acc *= q_scale;
    dqkv[(static_cast<long long>(b) * d.S + m) * d.ld_qkv + static_cast<long long>(which) * d.C + h * HD + c] =
        __float2bfloat16(acc);
  }
}


static int make_dims(AttnDims& d, int B, int H, int T, int L, int M, int C) {
  if (C != H * HD) return fail("vip_attention: head_dim must be 64 (C == 64*H)");
  if (L < 1) return fail("vip_attention: L must be >= 1");
  if (M < 1 || M > 8) return fail("vip_attention: 1 <= M <= 8 global tokens");
  d.B = B; d.H = H; d.T = T; d.L = L; d.M = M;
  d.S = static_cast<long long>(M) + static_cast<long long>(T) * L;
  d.C = C;
  d.ld_qkv = 3LL * C;
  d.ld_o = C;
  return 0;
}

// TMA maps of a [B*S, width] bf16 matrix: boxes of 64 columns x L frame rows and 64 columns x M global rows
static int make_row_maps(CUtensorMap* mL, CUtensorMap* mM, const void* base, long long width, const AttnDims& d) {
  const uint64_t rows = static_cast<uint64_t>(d.B) * static_cast<uint64_t>(d.S);
  if (make_tmap_bf16_2d(mL, base, width, rows, width, HD, d.L)) return -1;
  return make_tmap_bf16_2d(mM, base, width, rows, width, HD, d.M);
}

constexpr int FWD_SMEM = 3 * MAT_BYTES + 1024 + 64;
constexpr int BWD_SMEM = 4 * MAT_BYTES + 2 * SROWS * 4 + 1024 + 64;

}  // namespace xp

using namespace xp;

extern "C" int64_t xp_vip_attention_workspace_bytes(int32_t B, int32_t H, int32_t T, int32_t M) {
  // forward partials (66 floats) and backward partials (192 floats) per (b, h, t, m); sized for the larger
  return static_cast<int64_t>(B) * H * T * M * 3 * HD * sizeof(float);
}

extern "C" int xp_vip_attention_fwd(const void* qkv, void* out, float* lse, float* workspace, int32_t B, int32_t H,
                                    int32_t T, int32_t L, int32_t M, int32_t C, void* stream) {
  XP_ENTER(qkv);
  AttnDims d;
  if (make_dims(d, B, H, T, L, M, C)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (M + L > VIP_STAGED_MAX_ROWS) {   // frames too long to stage whole: the streamed kernel (vip_attention_long.cu)
    if (vip_long_attn_fwd(d, qkv, out, lse, workspace, st)) return -1;
  } else {
    CUtensorMap mL, mM;
    if (make_row_maps(&mL, &mM, qkv, 3LL * C, d)) return -1;
    if (smem_limit<vip_attn_fwd_kernel>(FWD_SMEM)) return -1;
    vip_attn_fwd_kernel<<<dim3(T, H, B), ATT_THREADS, FWD_SMEM, st>>>(mL, mM, static_cast<__nv_bfloat16*>(out), lse, workspace, d);
    XP_CHECK_LAUNCH("vip_attn_fwd_kernel");
  }
  vip_attn_fwd_combine_kernel<<<dim3(H, B), 64, 0, st>>>(workspace, static_cast<__nv_bfloat16*>(out), lse, d);
  XP_CHECK_LAUNCH("vip_attn_fwd_combine_kernel");
  return 0;
}

extern "C" int xp_vip_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                    float* workspace, int32_t B, int32_t H, int32_t T, int32_t L, int32_t M, int32_t C,
                                    float q_scale, void* stream) {
  XP_ENTER(qkv);
  AttnDims d;
  if (make_dims(d, B, H, T, L, M, C)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (M + L > VIP_STAGED_MAX_ROWS) {
    if (vip_long_attn_bwd(d, qkv, out, dout, lse, dqkv, workspace, q_scale, st)) return -1;
  } else {
    CUtensorMap mL, mM, gL, gM;
    if (make_row_maps(&mL, &mM, qkv, 3LL * C, d) || make_row_maps(&gL, &gM, dout, C, d)) return -1;
    if (smem_limit<vip_attn_bwd_kernel>(BWD_SMEM)) return -1;
    vip_attn_bwd_kernel<<<dim3(T, H, B), ATT_THREADS, BWD_SMEM, st>>>(
        mL, mM, gL, gM, static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), lse,
        static_cast<__nv_bfloat16*>(dqkv), workspace, d, q_scale);
    XP_CHECK_LAUNCH("vip_attn_bwd_kernel");
  }
  vip_attn_bwd_combine_kernel<<<dim3(H, B), 192, 0, st>>>(workspace, static_cast<__nv_bfloat16*>(dqkv), d, q_scale);
  XP_CHECK_LAUNCH("vip_attn_bwd_combine_kernel");
  return 0;
}
