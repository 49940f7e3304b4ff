// Strided, segmented multi-head attention (head_dim 64), forward and backward: the two attentions of HD-VILA's
// divided space-time TimeSformer block (BASELINE.json config #4).
//
// Reference: Attention.forward timesformer.py:156-173 called from Block.forward :207-222 on
//   temporal groups  'b (h w t) m -> (b h w) t m'   (T tokens, contiguous rows)            and
//   spatial groups   'b (h w t) m -> (b t) (h w) m' (H*W tokens, T rows apart).
// The reference materialises both rearranges (and their inverses) as copies; here the token-major [rows, 3C] qkv
// buffer never moves: a "sequence" is {first row, row stride, length}, and attention may be further restricted to
// segments of `seg` consecutive sequence positions (block-diagonal), which lets one CTA handle 64/T temporal groups
// at once instead of wasting a 64-row tile on 7 tokens.  q arrives pre-scaled by head_dim**-0.5 (QKV GEMM epilogue).
//
// Kernels (mma.sync.m16n8k16 bf16 -> fp32, flash-attention style, 4 warps x 16 rows per CTA, K/V or Q/dO streamed in
// 64-row blocks through a double-buffered cp.async ring):
//   seg_attn_fwd_kernel    online softmax, writes O (bf16) and the row log-sum-exp
//   seg_attn_delta_kernel  delta = rowsum(dO * O)
//   seg_attn_dkv_kernel    key-stationary:   dK, dV
//   seg_attn_dq_kernel     query-stationary: dQ (scaled back through the q pre-scale)
// The attentions are 0.5-2 % of a TimeSformer block's FLOPs (the wgmma GEMMs around them carry the rest).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "mma_frag.cuh"
#include "ptx.cuh"

namespace xp {

constexpr int SEG_BLK = 64;        // rows per staged block
constexpr int SEG_THREADS = 128;   // 4 warps x 16 rows
constexpr int SEG_TILE_BYTES = SEG_BLK * 128;

struct SegDev {
  long long n_rows, ld_qkv, ld_o, outer_stride, inner_stride, tok_stride;
  int H, C, n_seq, L, seg, inner;
  // window-attention extensions (LF-VILA Swin-3D, BASELINE.json config #5)
  const int* idx;          // [n_seq, L] token row of every sequence position (replaces the stride pattern) or nullptr
  const float* bias;       // [bias_nw, H, L, L] additive logits bias (relative-position bias + shift mask) or nullptr
  __nv_bfloat16* ds_out;   // dq kernel: [n_seq, H, L, L] dL/dlogits for the bias gradient, or nullptr
  int bias_nw;             // sequence s uses bias slab s % bias_nw
  int hd;                  // head dim 64 or 32 (32: rows are zero-padded to 64 columns in shared memory)
};

__device__ __forceinline__ long long seq_base(const SegDev& d, int s) {
  return static_cast<long long>(s / d.inner) * d.outer_stride + static_cast<long long>(s % d.inner) * d.inner_stride;
}
__device__ __forceinline__ int seq_len(const SegDev& d, long long base) {
  if (d.idx != nullptr) return d.L;
  const long long fit = (d.n_rows - base + d.tok_stride - 1) / d.tok_stride;
  return static_cast<int>(fit < d.L ? fit : d.L);
}

// Token row of position i of sequence s.
__device__ __forceinline__ long long tok_row(const SegDev& d, int s, long long base, int i) {
  return d.idx != nullptr ? static_cast<long long>(d.idx[static_cast<long long>(s) * d.L + i]) : base + i * d.tok_stride;
}
// Stage sequence positions [i0, i0+64) of one head slice (hd columns, zero-padded to 64) into a swizzled tile;
// positions >= len are zero.
__device__ __forceinline__ void stage_rows(uint32_t tile, const __nv_bfloat16* __restrict__ src, long long ld, const SegDev& d,
                                           int s, long long base, int i0, int len) {
  const int live_chunks = d.hd >> 3;
  for (int idx = threadIdx.x; idx < SEG_BLK * 8; idx += SEG_THREADS) {
    const int r = idx >> 3, chunk = idx & 7;
    const uint32_t dst = tile_addr(tile, r, chunk);
    const int i = i0 + r;
    if (i < len && chunk < live_chunks) cp_async16(dst, src + tok_row(d, s, base, i) * ld + chunk * 8);
    else st_shared_zero16(dst);
  }
}
// Additive logits bias of (sequence s, head h): row q, column key at bp[q * L + key].
__device__ __forceinline__ const float* bias_slab(const SegDev& d, int s, int h) {
  return d.bias + ((static_cast<long long>(s % d.bias_nw) * d.H + h) * d.L) * d.L;
}

// Block range [lo, hi) (in units of 64 positions) that can interact with positions [i0, i0+64) under the segment mask.
__device__ __forceinline__ void partner_blocks(const SegDev& d, int i0, int len, int& lo, int& hi) {
  if (d.seg >= d.L) {
    lo = 0;
    hi = (len + SEG_BLK - 1) / SEG_BLK;
    return;
  }
  const int last = min(i0 + SEG_BLK, len) - 1;
  const int p_lo = (i0 / d.seg) * d.seg;
  const int p_hi = min(len, (last / d.seg + 1) * d.seg);
  lo = p_lo / SEG_BLK;
  hi = (p_hi + SEG_BLK - 1) / SEG_BLK;
}

// ================================================================================ forward
// grid (ceil(L/64), H, n_seq)
template <int HDIM, bool BIAS>   // HDIM 64, or 32: half the k-steps and output column tiles; BIAS: additive logits slab
__global__ void __launch_bounds__(SEG_THREADS, HDIM == 32 ? 5 : 4)   // small windows are latency-bound: more resident CTAs
seg_attn_fwd_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                    const SegDev d) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sQ = (raw + 127u) & ~127u;
  const uint32_t sK0 = sQ + SEG_TILE_BYTES, sV0 = sK0 + 2 * SEG_TILE_BYTES;
  uint8_t* sQ_ptr = smem_raw + (sQ - raw);
  const int h = blockIdx.y, s = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long base = seq_base(d, s);
  if (d.idx == nullptr && base >= d.n_rows) return;
  const int len = seq_len(d, base);
  const int q0 = blockIdx.x * SEG_BLK;
  if (q0 >= len) return;
  int kb_lo, kb_hi;
  partner_blocks(d, q0, len, kb_lo, kb_hi);
  const __nv_bfloat16* qsrc = qkv + h * d.hd;
  const __nv_bfloat16* ksrc = qsrc + d.C;
  const __nv_bfloat16* vsrc = qsrc + 2 * d.C;

  stage_rows(sQ, qsrc, d.ld_qkv, d, s, base, q0, len);
  stage_rows(sK0, ksrc, d.ld_qkv, d, s, base, kb_lo * SEG_BLK, len);
  stage_rows(sV0, vsrc, d.ld_qkv, d, s, base, kb_lo * SEG_BLK, len);
  cp_async_commit();

  uint32_t qa[4][4];
  constexpr int KS = HDIM / 16, ND = HDIM / 8;
  float o[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int row_lo = q0 + warp * 16 + (lane >> 2);   // this thread's rows: row_lo, row_lo + 8
  int seg_lo[2], seg_hi[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = row_lo + r * 8;
    seg_lo[r] = d.seg >= d.L ? 0 : (q / d.seg) * d.seg;
    seg_hi[r] = d.seg >= d.L ? len : min(len, seg_lo[r] + d.seg);
  }

  for (int kb = kb_lo; kb < kb_hi; ++kb) {
    const int buf = (kb - kb_lo) & 1;
    if (kb + 1 < kb_hi) {
      stage_rows(sK0 + (buf ^ 1) * SEG_TILE_BYTES, ksrc, d.ld_qkv, d, s, base, (kb + 1) * SEG_BLK, len);
      stage_rows(sV0 + (buf ^ 1) * SEG_TILE_BYTES, vsrc, d.ld_qkv, d, s, base, (kb + 1) * SEG_BLK, len);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kb == kb_lo) load_a_frags(sQ, warp * 16, lane, qa);
    const uint32_t sK = sK0 + buf * SEG_TILE_BYTES, sV = sV0 + buf * SEG_TILE_BYTES;
    const int key0 = kb * SEG_BLK;

    float sc[8][4];
    const float* bp = BIAS ? bias_slab(d, s, h) : nullptr;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // accumulators start at the additive bias: its loads overlap the Q K^T MMAs
        const int key = key0 + i * 8 + (lane & 3) * 2 + (e & 1);
        const int q = row_lo + (e >> 1) * 8;
        sc[i][e] = (BIAS && key < len && q < len) ? bp[static_cast<long long>(q) * d.L + key] : 0.f;
      }
    }
#pragma unroll
    for (int np = 0; np < 4; ++np) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t b[4];
        load_b_nk(sK, np * 16, ks, lane, b);
        mma_bf16(sc[2 * np], qa[ks], b[0], b[1]);
        mma_bf16(sc[2 * np + 1], qa[ks], b[2], b[3]);
      }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = key0 + i * 8 + (lane & 3) * 2 + (e & 1);
        const int r = e >> 1;
        if (key < seg_lo[r] || key >= seg_hi[r]) sc[i][e] = -INFINITY;
        mx[r] = fmaxf(mx[r], sc[i][e]);
      }
    }
    float corr[2], m_new[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      m_new[r] = fmaxf(m_run[r], mx[r]);
      corr[r] = (m_new[r] == -INFINITY) ? 1.f : fast_exp2((m_run[r] - m_new[r]) * LOG2E);
      l_run[r] *= corr[r];
      m_run[r] = m_new[r];
    }
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    const float mb[2] = {m_new[0] == -INFINITY ? 0.f : m_new[0] * LOG2E, m_new[1] == -INFINITY ? 0.f : m_new[1] * LOG2E};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = fast_exp2(fmaf(sc[i][e], LOG2E, -mb[e >> 1]));   // exp2(-inf) = 0 for masked entries
        sc[i][e] = pv;
        l_run[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      pa[0] = pack_bf16(sc[2 * kk][0], sc[2 * kk][1]);
      pa[1] = pack_bf16(sc[2 * kk][2], sc[2 * kk][3]);
      pa[2] = pack_bf16(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
      pa[3] = pack_bf16(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < KS; ++dp) {
        uint32_t b[4];
        load_b_kn(sV, kk * 16, dp, lane, b);
        mma_bf16(o[2 * dp], pa, b[0], b[1]);
        mma_bf16(o[2 * dp + 1], pa, b[2], b[3]);
      }
    }
    __syncthreads();   // every warp is done with this buffer before the next iteration refills it
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
  // normalise, stage through this warp's (dead) Q rows, store 128-byte rows
#pragma unroll
  for (int i = 0; i < ND; ++i) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = warp * 16 + (lane >> 2) + r * 8;
      const uint32_t v = pack_bf16(o[i][2 * r] * inv[r], o[i][2 * r + 1] * inv[r]);
      *reinterpret_cast<uint32_t*>(sQ_ptr + (tile_addr(sQ, row, i) - sQ) + (lane & 3) * 4) = v;
    }
  }
  __syncwarp();
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int idx = lane + it * 32;
    const int row = warp * 16 + (idx >> 3), chunk = idx & 7;
    if (q0 + row < len && chunk < (d.hd >> 3)) {
      const uint4 v = *reinterpret_cast<const uint4*>(sQ_ptr + (tile_addr(sQ, row, chunk) - sQ));
      *reinterpret_cast<uint4*>(out + tok_row(d, s, base, q0 + row) * d.ld_o + h * d.hd + chunk * 8) = v;
    }
  }
  if ((lane & 3) == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = row_lo + r * 8;
      if (q < len) lse[static_cast<long long>(h) * d.n_rows + tok_row(d, s, base, q)] = m_run[r] + logf(l_run[r]);
    }
  }
}

// ================================================================================ delta = rowsum(dO * O)
// 8 lanes per (row, head); delta: [H, n_rows]
__global__ void __launch_bounds__(256)
seg_attn_delta_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                      float* __restrict__ delta, long long n_rows, int H, long long ld_o, int hd) {
  const long long gid = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  const long long item = gid >> 3;
  const int chunk = gid & 7;
  const bool live = item < n_rows * H && chunk < (hd >> 3);
  float dot = 0.f;
  long long row = 0;
  int h = 0;
  if (item < n_rows * H) {
    row = item / H;
    h = static_cast<int>(item - row * H);
  }
  if (live) {
    const long long off = row * ld_o + h * hd + chunk * 8;
    const uint4 g = *reinterpret_cast<const uint4*>(dout + off);
    const uint4 o = *reinterpret_cast<const uint4*>(out + off);
    const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) dot += bf16_lo(gw[i]) * bf16_lo(ow[i]) + bf16_hi(gw[i]) * bf16_hi(ow[i]);
  }
  dot += __shfl_xor_sync(0xffffffffu, dot, 1);
  dot += __shfl_xor_sync(0xffffffffu, dot, 2);
  dot += __shfl_xor_sync(0xffffffffu, dot, 4);
  if (item < n_rows * H && chunk == 0) delta[static_cast<long long>(h) * n_rows + row] = dot;
}

// Stage lse * log2(e) (+inf on padding, so p = exp2(s - inf) = 0) and delta of positions [i0, i0+64).
__device__ __forceinline__ void stage_stats(float* s_lse, float* s_delta, const float* __restrict__ lse,
                                            const float* __restrict__ delta, const SegDev& d, int s, int h, long long base,
                                            int i0, int len) {
  if (threadIdx.x < SEG_BLK) {
    const int i = i0 + threadIdx.x;
    const long long at = static_cast<long long>(h) * d.n_rows + (i < len ? tok_row(d, s, base, i) : 0);
    s_lse[threadIdx.x] = i < len ? lse[at] * LOG2E : INFINITY;
    s_delta[threadIdx.x] = i < len ? delta[at] : 0.f;
  }
}

// ================================================================================ backward: dK, dV
// grid (ceil(L/64) key blocks, H, n_seq); each warp keeps 16 keys' K, V fragments and dK, dV accumulators in registers
// and streams the query blocks (Q, dO, lse, delta) through shared memory.
template <int HDIM, bool BIAS>
__global__ void __launch_bounds__(SEG_THREADS, HDIM == 32 ? 4 : 3)
seg_attn_dkv_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout,
                    const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                    const SegDev d) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sK = (raw + 127u) & ~127u;
  const uint32_t sV = sK + SEG_TILE_BYTES, sQ0 = sV + SEG_TILE_BYTES, sdO0 = sQ0 + 2 * SEG_TILE_BYTES;
  float* s_lse0 = reinterpret_cast<float*>(smem_raw + (sdO0 + 2 * SEG_TILE_BYTES - raw));
  float* s_delta0 = s_lse0 + 2 * SEG_BLK;
  const int h = blockIdx.y, s = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long base = seq_base(d, s);
  if (d.idx == nullptr && base >= d.n_rows) return;
  const int len = seq_len(d, base);
  const int k0 = blockIdx.x * SEG_BLK;
  if (k0 >= len) return;
  int qb_lo, qb_hi;
  partner_blocks(d, k0, len, qb_lo, qb_hi);
  const __nv_bfloat16* qsrc = qkv + h * d.hd;
  const __nv_bfloat16* dosrc = dout + h * d.hd;

  stage_rows(sK, qsrc + d.C, d.ld_qkv, d, s, base, k0, len);
  stage_rows(sV, qsrc + 2 * d.C, d.ld_qkv, d, s, base, k0, len);
  stage_rows(sQ0, qsrc, d.ld_qkv, d, s, base, qb_lo * SEG_BLK, len);
  stage_rows(sdO0, dosrc, d.ld_o, d, s, base, qb_lo * SEG_BLK, len);
  cp_async_commit();
  stage_stats(s_lse0, s_delta0, lse, delta, d, s, h, base, qb_lo * SEG_BLK, len);

  uint32_t ka[4][4], va[4][4];
  constexpr int KS = HDIM / 16, ND = HDIM / 8;
  float dk[ND][4], dv[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  const int key_lo = k0 + warp * 16 + (lane >> 2);
  int seg_lo[2], seg_hi[2];
  bool key_ok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_lo + r * 8;
    key_ok[r] = key < len;
    seg_lo[r] = d.seg >= d.L ? 0 : (key / d.seg) * d.seg;
    seg_hi[r] = d.seg >= d.L ? len : min(len, seg_lo[r] + d.seg);
  }

  const float* bp = BIAS ? bias_slab(d, s, h) : nullptr;
  for (int qb = qb_lo; qb < qb_hi; ++qb) {
    const int buf = (qb - qb_lo) & 1;
    if (qb + 1 < qb_hi) {
      stage_rows(sQ0 + (buf ^ 1) * SEG_TILE_BYTES, qsrc, d.ld_qkv, d, s, base, (qb + 1) * SEG_BLK, len);
      stage_rows(sdO0 + (buf ^ 1) * SEG_TILE_BYTES, dosrc, d.ld_o, d, s, base, (qb + 1) * SEG_BLK, len);
      cp_async_commit();
      stage_stats(s_lse0 + (buf ^ 1) * SEG_BLK, s_delta0 + (buf ^ 1) * SEG_BLK, lse, delta, d, s, h, base, (qb + 1) * SEG_BLK, len);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (qb == qb_lo) {
      load_a_frags(sK, warp * 16, lane, ka);
      load_a_frags(sV, warp * 16, lane, va);
    }
    const uint32_t sQ = sQ0 + buf * SEG_TILE_BYTES, sdO = sdO0 + buf * SEG_TILE_BYTES;
    const float* s_lse = s_lse0 + buf * SEG_BLK;
    const float* s_delta = s_delta0 + buf * SEG_BLK;
    const int qbase = qb * SEG_BLK;
#pragma unroll 1
    for (int sub = 0; sub < 4; ++sub) {
      if (qbase + sub * 16 >= len) break;
      float st[2][4], dpt[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // S^T accumulators start at the additive bias (loads overlap the MMAs)
          const int q = qbase + sub * 16 + i * 8 + (lane & 3) * 2 + (e & 1);
          const int key = key_lo + (e >> 1) * 8;
          st[i][e] = (BIAS && q < len && key < len) ? bp[static_cast<long long>(q) * d.L + key] : 0.f;
        }
      }
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t bq[4], bo[4];
        load_b_nk(sQ, sub * 16, ks, lane, bq);
        load_b_nk(sdO, sub * 16, ks, lane, bo);
        mma_bf16(st[0], ka[ks], bq[0], bq[1]);
        mma_bf16(st[1], ka[ks], bq[2], bq[3]);
        mma_bf16(dpt[0], va[ks], bo[0], bo[1]);
        mma_bf16(dpt[1], va[ks], bo[2], bo[3]);
      }
      float pt[2][4], dst[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int ql = sub * 16 + i * 8 + (lane & 3) * 2 + (e & 1);   // query within the staged block
          const int q = qbase + ql;
          const int r = e >> 1;
          const bool valid = key_ok[r] && q >= seg_lo[r] && q < seg_hi[r];
          const float p = valid ? fast_exp2(fmaf(st[i][e], LOG2E, -s_lse[ql])) : 0.f;
          pt[i][e] = p;
          dst[i][e] = p * (dpt[i][e] - s_delta[ql]);
        }
      }
      uint32_t pa[4], da[4];
      pa[0] = pack_bf16(pt[0][0], pt[0][1]); pa[1] = pack_bf16(pt[0][2], pt[0][3]);
      pa[2] = pack_bf16(pt[1][0], pt[1][1]); pa[3] = pack_bf16(pt[1][2], pt[1][3]);
      da[0] = pack_bf16(dst[0][0], dst[0][1]); da[1] = pack_bf16(dst[0][2], dst[0][3]);
      da[2] = pack_bf16(dst[1][0], dst[1][1]); da[3] = pack_bf16(dst[1][2], dst[1][3]);
#pragma unroll
      for (int dp = 0; dp < KS; ++dp) {
        uint32_t bo[4], bq[4];
        load_b_kn(sdO, sub * 16, dp, lane, bo);
        load_b_kn(sQ, sub * 16, dp, lane, bq);
        mma_bf16(dv[2 * dp], pa, bo[0], bo[1]);
        mma_bf16(dv[2 * dp + 1], pa, bo[2], bo[3]);
        mma_bf16(dk[2 * dp], da, bq[0], bq[1]);
        mma_bf16(dk[2 * dp + 1], da, bq[2], bq[3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = key_lo + r * 8;
    if (key >= len) continue;
    __nv_bfloat16* row = dqkv + tok_row(d, s, base, key) * d.ld_qkv + h * d.hd + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      *reinterpret_cast<uint32_t*>(row + d.C + i * 8) = pack_bf16(dk[i][2 * r], dk[i][2 * r + 1]);
      *reinterpret_cast<uint32_t*>(row + 2 * d.C + i * 8) = pack_bf16(dv[i][2 * r], dv[i][2 * r + 1]);
    }
  }
}

// ================================================================================ backward: dQ
// grid (ceil(L/64) query blocks, H, n_seq); Q, dO fragments + dQ accumulators in registers, K/V blocks streamed.
template <int HDIM, bool BIAS>
__global__ void __launch_bounds__(SEG_THREADS, HDIM == 32 ? 5 : 4)
seg_attn_dq_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ dout,
                   const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                   const SegDev d, float q_scale) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sQ = (raw + 127u) & ~127u;
  const uint32_t sdO = sQ + SEG_TILE_BYTES, sK0 = sdO + SEG_TILE_BYTES, sV0 = sK0 + 2 * SEG_TILE_BYTES;
  const int h = blockIdx.y, s = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long base = seq_base(d, s);
  if (d.idx == nullptr && base >= d.n_rows) return;
  const int len = seq_len(d, base);
  const int q0 = blockIdx.x * SEG_BLK;
  if (q0 >= len) return;
  int kb_lo, kb_hi;
  partner_blocks(d, q0, len, kb_lo, kb_hi);
  const __nv_bfloat16* qsrc = qkv + h * d.hd;
  const __nv_bfloat16* ksrc = qsrc + d.C;
  const __nv_bfloat16* vsrc = qsrc + 2 * d.C;

  stage_rows(sQ, qsrc, d.ld_qkv, d, s, base, q0, len);
  stage_rows(sdO, dout + h * d.hd, d.ld_o, d, s, base, q0, len);
  stage_rows(sK0, ksrc, d.ld_qkv, d, s, base, kb_lo * SEG_BLK, len);
  stage_rows(sV0, vsrc, d.ld_qkv, d, s, base, kb_lo * SEG_BLK, len);
  cp_async_commit();

  uint32_t qa[4][4], oa[4][4];
  constexpr int KS = HDIM / 16, ND = HDIM / 8;
  float dq[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const int q_lo = q0 + warp * 16 + (lane >> 2);
  float lse_r[2], del_r[2];
  int seg_lo[2], seg_hi[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q_lo + r * 8;
    const long long at = static_cast<long long>(h) * d.n_rows + (q < len ? tok_row(d, s, base, q) : 0);
    lse_r[r] = q < len ? lse[at] * LOG2E : INFINITY;
    del_r[r] = q < len ? delta[at] : 0.f;
    seg_lo[r] = d.seg >= d.L ? 0 : (q / d.seg) * d.seg;
    seg_hi[r] = d.seg >= d.L ? len : min(len, seg_lo[r] + d.seg);
  }

  const float* bp = BIAS ? bias_slab(d, s, h) : nullptr;
  __nv_bfloat16* dsp = d.ds_out != nullptr ? d.ds_out + ((static_cast<long long>(s) * d.H + h) * d.L) * d.L : nullptr;
  for (int kb = kb_lo; kb < kb_hi; ++kb) {
    const int buf = (kb - kb_lo) & 1;
    if (kb + 1 < kb_hi) {
      stage_rows(sK0 + (buf ^ 1) * SEG_TILE_BYTES, ksrc, d.ld_qkv, d, s, base, (kb + 1) * SEG_BLK, len);
      stage_rows(sV0 + (buf ^ 1) * SEG_TILE_BYTES, vsrc, d.ld_qkv, d, s, base, (kb + 1) * SEG_BLK, len);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kb == kb_lo) {
      load_a_frags(sQ, warp * 16, lane, qa);
      load_a_frags(sdO, warp * 16, lane, oa);
    }
    const uint32_t sK = sK0 + buf * SEG_TILE_BYTES, sV = sV0 + buf * SEG_TILE_BYTES;
    const int kbase = kb * SEG_BLK;
#pragma unroll 1
    for (int sub = 0; sub < 4; ++sub) {
      if (kbase + sub * 16 >= len) break;
      float sc[2][4], dp_[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {   // logits accumulators start at the additive bias (loads overlap the MMAs)
          const int key = kbase + sub * 16 + i * 8 + (lane & 3) * 2 + (e & 1);
          const int q = q_lo + (e >> 1) * 8;
          sc[i][e] = (BIAS && q < len && key < len) ? bp[static_cast<long long>(q) * d.L + key] : 0.f;
        }
      }
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        uint32_t bk[4], bv[4];
        load_b_nk(sK, sub * 16, ks, lane, bk);
        load_b_nk(sV, sub * 16, ks, lane, bv);
        mma_bf16(sc[0], qa[ks], bk[0], bk[1]);
        mma_bf16(sc[1], qa[ks], bk[2], bk[3]);
        mma_bf16(dp_[0], oa[ks], bv[0], bv[1]);
        mma_bf16(dp_[1], oa[ks], bv[2], bv[3]);
      }
      float ds[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = kbase + sub * 16 + i * 8 + (lane & 3) * 2 + (e & 1);
          const int r = e >> 1;
          const bool valid = key >= seg_lo[r] && key < seg_hi[r];
          const int q = q_lo + r * 8;
          const float p = valid ? fast_exp2(fmaf(sc[i][e], LOG2E, -lse_r[r])) : 0.f;
          ds[i][e] = p * (dp_[i][e] - del_r[r]);
          if (BIAS && dsp != nullptr && q < len && key < len) dsp[static_cast<long long>(q) * d.L + key] = __float2bfloat16(ds[i][e]);
        }
      }
      uint32_t da[4];
      da[0] = pack_bf16(ds[0][0], ds[0][1]); da[1] = pack_bf16(ds[0][2], ds[0][3]);
      da[2] = pack_bf16(ds[1][0], ds[1][1]); da[3] = pack_bf16(ds[1][2], ds[1][3]);
#pragma unroll
      for (int dp = 0; dp < KS; ++dp) {
        uint32_t bk[4];
        load_b_kn(sK, sub * 16, dp, lane, bk);
        mma_bf16(dq[2 * dp], da, bk[0], bk[1]);
        mma_bf16(dq[2 * dp + 1], da, bk[2], bk[3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q_lo + r * 8;
    if (q >= len) continue;
    __nv_bfloat16* row = dqkv + tok_row(d, s, base, q) * d.ld_qkv + h * d.hd + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < ND; ++i) {
      *reinterpret_cast<uint32_t*>(row + i * 8) = pack_bf16(dq[i][2 * r] * q_scale, dq[i][2 * r + 1] * q_scale);
    }
  }
}

constexpr const char* SEG_BAD_HD = "xp_seg_attention: head_dim must be 64 (or 0) or 32";

static int to_dev(const XpSegAttn* a, SegDev& d, const char* who) {
  if (a == nullptr) return fail("xp_seg_attention: null descriptor");
  if (a->heads <= 0 || a->n_rows <= 0 || a->n_seq <= 0 || a->seq_len <= 0 || a->seg_len <= 0 || a->inner <= 0 ||
      a->tok_stride <= 0)
    return fail("xp_seg_attention: heads, n_rows, n_seq, seq_len, seg_len, inner and tok_stride must be positive");
  d.hd = a->head_dim == 0 ? HD : a->head_dim;
  if (d.hd != 64 && d.hd != 32) return fail(SEG_BAD_HD);
  d.H = a->heads;
  d.C = a->heads * d.hd;
  d.idx = a->row_index;
  d.bias = a->bias;
  d.bias_nw = a->bias_windows > 0 ? a->bias_windows : 1;
  d.ds_out = static_cast<__nv_bfloat16*>(a->ds_out);
  if (d.idx != nullptr && a->seg_len < a->seq_len) return fail("xp_seg_attention: row_index sequences are dense (seg_len >= seq_len)");
  if (a->ld_qkv < 3LL * d.C || a->ld_out < d.C || a->ld_qkv % 8 || a->ld_out % 8)
    return fail("xp_seg_attention: ld_qkv >= 3*heads*64, ld_out >= heads*64, both multiples of 8");
  d.n_rows = a->n_rows; d.ld_qkv = a->ld_qkv; d.ld_o = a->ld_out;
  d.outer_stride = a->outer_stride; d.inner_stride = a->inner_stride; d.tok_stride = a->tok_stride;
  d.n_seq = a->n_seq; d.L = a->seq_len; d.seg = a->seg_len; d.inner = a->inner;
  (void)who;
  return 0;
}

constexpr int SEG_FWD_SMEM = 5 * SEG_TILE_BYTES + 128;
constexpr int SEG_DKV_SMEM = 6 * SEG_TILE_BYTES + 4 * SEG_BLK * 4 + 128;
constexpr int SEG_DQ_SMEM = 6 * SEG_TILE_BYTES + 128;

}  // namespace xp

using namespace xp;

// grid (64-row blocks, heads, sequences); the z limit of 65535 sequences is checked by the callers below
static dim3 seg_grid(const SegDev& d) { return dim3((d.L + SEG_BLK - 1) / SEG_BLK, d.H, d.n_seq); }

// f(head_dim, with_bias) as template arguments; to_dev has refused every other head_dim
template <class F>
static int seg_dispatch(const SegDev& d, F&& f) {
  return dispatch<64, 32>(d.hd, SEG_BAD_HD, [&](auto hd) {
    return dispatch<0, 1>(d.bias != nullptr, SEG_BAD_HD, [&](auto b) { return f(hd, b); });
  });
}

extern "C" int xp_seg_attention_fwd(const void* qkv, void* out, float* lse, const XpSegAttn* desc, void* stream) {
  XP_ENTER(qkv);
  SegDev d;
  if (int rc = to_dev(desc, d, "fwd")) return rc;
  if (d.n_seq > 65535) return fail("xp_seg_attention_fwd: n_seq > 65535 (split the call)");
  return seg_dispatch(d, [&](auto hd, auto b) {
    constexpr auto kern = seg_attn_fwd_kernel<hd.value, b.value>;
    if (smem_limit<kern>(SEG_FWD_SMEM)) return -1;
    kern<<<seg_grid(d), SEG_THREADS, SEG_FWD_SMEM, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(out), lse, d);
    XP_CHECK_LAUNCH("seg_attn_fwd_kernel");
    return 0;
  });
}

extern "C" int xp_seg_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                                    void* dqkv, const XpSegAttn* desc, float q_scale, void* stream) {
  XP_ENTER(qkv);
  SegDev d;
  if (int rc = to_dev(desc, d, "bwd")) return rc;
  if (d.n_seq > 65535) return fail("xp_seg_attention_bwd: n_seq > 65535 (split the call)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __nv_bfloat16* qp = static_cast<const __nv_bfloat16*>(qkv);
  const __nv_bfloat16* dop = static_cast<const __nv_bfloat16*>(dout);
  __nv_bfloat16* dqp = static_cast<__nv_bfloat16*>(dqkv);
  return seg_dispatch(d, [&](auto hd, auto b) {
    constexpr auto dkv = seg_attn_dkv_kernel<hd.value, b.value>;
    constexpr auto dq = seg_attn_dq_kernel<hd.value, b.value>;
    if (smem_limit<dkv>(SEG_DKV_SMEM) || smem_limit<dq>(SEG_DQ_SMEM)) return -1;
    const long long items = d.n_rows * d.H * 8;
    seg_attn_delta_kernel<<<static_cast<unsigned>((items + 255) / 256), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), delta, d.n_rows, d.H, d.ld_o, d.hd);
    XP_CHECK_LAUNCH("seg_attn_delta_kernel");
    dkv<<<seg_grid(d), SEG_THREADS, SEG_DKV_SMEM, st>>>(qp, dop, lse, delta, dqp, d);
    XP_CHECK_LAUNCH("seg_attn_dkv_kernel");
    dq<<<seg_grid(d), SEG_THREADS, SEG_DQ_SMEM, st>>>(qp, dop, lse, delta, dqp, d, q_scale);
    XP_CHECK_LAUNCH("seg_attn_dq_kernel");
    return 0;
  });
}
