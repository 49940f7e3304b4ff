// Video-proxy (ViP) attention for frames longer than the staged kernel of vip_attention.cu takes (M + L > 208): ViT-L/14
// has L = 256 patches per frame at 224 px, 576 at 336 px and 1024 at 448 px.  Same maths (CLIPAttention.forward2,
// CLIP_ViP.py:332-381), same outputs and the same per-frame partials of the global rows as vip_attention.cu, whose combine
// kernels finish both paths.
//
// A frame is too long to stage whole (a TMA box holds at most 256 rows), so K / V (backward: Q / dO) are streamed.  The
// rows of one (b, h, t) are cut into tiles of 64: tiles j < nft = ceil(L / 64) hold frame rows [64 j, 64 j + 64) (rows
// past L are masked; TMA reads whatever follows, or zero fill at the end of the tensor), and tile nft holds the M global
// rows (rows past M masked).  Patch queries of frame t see every key tile of frame t plus the global tile; global queries
// see the same keys, except that the global keys count only in frame 0, so that global x global pairs enter once.
//
// Hopper path, FlashAttention-3 shaped: a CTA of three warpgroups per two 64-row tiles of one (b, h, t).  Warpgroup 0 is
// the producer (setmaxnreg down to 40): one thread streams 64-row blocks by TMA into 128B-swizzled shared memory
// through a two-stage full / empty mbarrier ring.  Warpgroups 1 and 2 are consumers (setmaxnreg up to 232), each owning
// one tile, with every product on wgmma:
//   forward    query-stationary: S = Q·Kᵀ, online softmax over the 64-key blocks in registers, O += P·V with P in
//              registers, split into bf16 hi + lo as in vip_attention.cu;
//   backward   key-stationary kernel: Sᵀ = K·Qᵀ and dPᵀ = V·dOᵀ per streamed query block, dV += Pᵀ·dO, dK += dSᵀ·Q; the
//              producer warpgroup also computes each block's delta = rowsum(dO * O) and loads its LSE.
//              query-stationary kernel: S = Q·Kᵀ and dP = dO·Vᵀ per streamed key block, dQ += dS·K.
// Every output element and every partial has exactly one writer and no float atomics are used, so results do not depend
// on scheduling.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"
#include "mma_frag.cuh"
#include "vip_attention.h"

namespace xp {

namespace {

constexpr int LTILE = 64;                   // rows per tile / streamed block
constexpr int LTILE_BYTES = LTILE * 128;    // one [64][64] bf16 tile, 128B-swizzled
constexpr int LONG_THREADS = 384;           // producer warpgroup + two consumer warpgroups
constexpr int LSTAGES = 2;                  // ring depth of the streamed blocks

__device__ __forceinline__ uint64_t kdesc(uint32_t addr) { return make_smem_desc_sw128(addr, 16, 1024); }     // K-major
__device__ __forceinline__ uint64_t mndesc(uint32_t addr) { return make_smem_desc_sw128(addr, 8192, 1024); }  // MN-major

__device__ __forceinline__ int num_frame_tiles(const AttnDims& d) { return (d.L + LTILE - 1) / LTILE; }
// first qkv / out row of tile j of (b, t): TMA row coordinate
__device__ __forceinline__ int tile_row0(const AttnDims& d, int nft, int b, int t, int j) {
  return static_cast<int>(static_cast<long long>(b) * d.S +
                          (j < nft ? d.M + static_cast<long long>(t) * d.L + static_cast<long long>(j) * LTILE : 0));
}
// live rows of tile j
__device__ __forceinline__ int tile_rows(const AttnDims& d, int nft, int j) {
  return j < nft ? min(LTILE, d.L - j * LTILE) : d.M;
}
// sequence index (within the sample) of row i of tile j
__device__ __forceinline__ long long tile_seq(const AttnDims& d, int nft, int t, int j, int i) {
  return j < nft ? d.M + static_cast<long long>(t) * d.L + static_cast<long long>(j) * LTILE + i : i;
}
// keys of key tile kb that the queries of query tile qt see: a prefix of the tile (0: skip the block)
__device__ __forceinline__ int live_keys(const AttnDims& d, int nft, int t, int qt, int kb) {
  if (kb < nft) return min(LTILE, d.L - kb * LTILE);
  return (qt == nft && t != 0) ? 0 : d.M;
}

__device__ __forceinline__ void acc_to_afrag(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16(x[8 * ks + 0], x[8 * ks + 1]);
    a[ks][1] = pack_bf16(x[8 * ks + 2], x[8 * ks + 3]);
    a[ks][2] = pack_bf16(x[8 * ks + 4], x[8 * ks + 5]);
    a[ks][3] = pack_bf16(x[8 * ks + 6], x[8 * ks + 7]);
  }
}

// delta = sum_c dO[row, c] * O[row, c] over a 16-column quarter (bf16 products in fp32)
__device__ __forceinline__ float dot16(const __nv_bfloat16* g, const __nv_bfloat16* o) {
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint4 gv = *reinterpret_cast<const uint4*>(g + 8 * j), ov = *reinterpret_cast<const uint4*>(o + 8 * j);
    const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w}, ow[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) acc += bf16_lo(gw[i]) * bf16_lo(ow[i]) + bf16_hi(gw[i]) * bf16_hi(ow[i]);
  }
  return acc;
}

// Barrier set-up of the ring; `full_count` arrivals complete a fill, every live consumer warp releases a stage.
__device__ __forceinline__ void init_ring(uint64_t* q_full, uint64_t* full, uint64_t* empty, uint32_t full_count,
                                          int nlive, const CUtensorMap* tm0, const CUtensorMap* tm1) {
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tm0);
    tma_prefetch_desc(tm1);
    mbar_init(q_full, 1);
#pragma unroll
    for (int s = 0; s < LSTAGES; ++s) {
      mbar_init(&full[s], full_count);
      mbar_init(&empty[s], 4 * nlive);
    }
    fence_barrier_init();
  }
  __syncthreads();
}
__device__ __forceinline__ void release_stage(uint64_t* empty, int s) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[s]);
}

}  // namespace

// ======================================================================== forward
// grid (ceil((nft + 1) / 2), T, B*H); consumer c of CTA x owns query tile 2x + c.  Shared memory: the two Q tiles, then
// LSTAGES x {K, V}.  Outputs as vip_attn_fwd_kernel.
__global__ void __launch_bounds__(LONG_THREADS, 1)
vip_long_fwd_kernel(const __grid_constant__ CUtensorMap tm, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                    float* __restrict__ part, const AttnDims d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (2 + 2 * LSTAGES) * LTILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + LSTAGES;
  const int t = blockIdx.y, h = blockIdx.z % d.H, b = blockIdx.z / d.H;
  const int nft = num_frame_tiles(d), ntiles = nft + 1;
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1, nlive, &tm, &tm);

  if (wg == 0) {
    // ------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * LTILE_BYTES);
      for (int c = 0; c < nlive; ++c) tma_load_2d(sm + c * LTILE_BYTES, &tm, q_full, h * HD, tile_row0(d, nft, b, t, qt0 + c));
      for (int kb = 0; kb < ntiles; ++kb) {
        const int s = kb % LSTAGES;
        mbar_wait_nocall(&empty[s], ((kb / LSTAGES) & 1) ^ 1);
        uint8_t* st = sm + (2 + 2 * s) * LTILE_BYTES;
        const int r0 = tile_row0(d, nft, b, t, kb);
        mbar_arrive_expect_tx(&full[s], 2 * LTILE_BYTES);
        tma_load_2d(st, &tm, &full[s], d.C + h * HD, r0);
        tma_load_2d(st + LTILE_BYTES, &tm, &full[s], 2 * d.C + h * HD, r0);
      }
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const bool qglob = qt == nft;
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int r_lo = wq * 16 + (lane >> 2);
  const uint32_t sQ = smem_u32(sm) + c * LTILE_BYTES;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % LSTAGES;
    const int klim = live_keys(d, nft, t, qt, kb);
    mbar_wait_nocall(&full[s], (kb / LSTAGES) & 1);
    if (klim == 0) {
      release_stage(empty, s);
      continue;
    }
    const uint32_t sK = smem_u32(sm) + (2 + 2 * s) * LTILE_BYTES, sV = sK + LTILE_BYTES;
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
    wgmma_fence_regs(sc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0, 0>(sc, kdesc(sQ + ks * 32), kdesc(sK + ks * 32));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = i * 8 + (lane & 3) * 2 + (e & 1);
        if (key >= klim) sc[4 * i + e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], sc[4 * i + e]);
      }
    float corr[2], mb[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      corr[r] = (m_new == -INFINITY) ? 1.f : fast_exp2((m_run[r] - m_new) * LOG2E);
      l_run[r] *= corr[r];
      m_run[r] = m_new;
      mb[r] = m_new == -INFINITY ? 0.f : m_new * LOG2E;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i + 0] *= corr[0]; o[4 * i + 1] *= corr[0];
      o[4 * i + 2] *= corr[1]; o[4 * i + 3] *= corr[1];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float pv = fast_exp2(fmaf(sc[i], LOG2E, -mb[(i >> 1) & 1]));   // exp2(-inf) = 0 for masked entries
      sc[i] = pv;
      l_run[(i >> 1) & 1] += pv;
    }
    // P·V with P = hi + lo in bf16 (vip_attention.cu: rounding P is the largest error and reaches the CLS features)
    uint32_t ph[4][4], pl[4][4];
    acc_to_afrag(sc, ph);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        pl[ks][j] = pack_bf16(sc[8 * ks + 2 * j] - bf16_lo(ph[ks][j]), sc[8 * ks + 2 * j + 1] - bf16_hi(ph[ks][j]));
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t vd = mndesc(sV + ks * 16 * 128);
      wgmma_m64n64k16_rs<1>(o, ph[ks], vd);
      wgmma_m64n64k16_rs<1>(o, pl[ks], vd);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    release_stage(empty, s);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const int qrows = tile_rows(d, nft, qt);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r_lo + r * 8;
    if (row >= qrows) continue;
    if (qglob) {   // global-query row: this frame's partial (fp32, unnormalised)
      float* p = part + (((static_cast<long long>(b) * d.H + h) * d.T + t) * d.M + row) * 66;
      if ((lane & 3) == 0) {
        p[0] = m_run[r];
        p[1] = l_run[r];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        p[2 + i * 8 + (lane & 3) * 2] = o[4 * i + 2 * r];
        p[2 + i * 8 + (lane & 3) * 2 + 1] = o[4 * i + 2 * r + 1];
      }
    } else {       // frame row: normalised output + LSE
      const float inv = l_run[r] > 0.f ? 1.f / l_run[r] : 0.f;
      const long long seq = tile_seq(d, nft, t, qt, row);
      __nv_bfloat16* dst = out + (static_cast<long long>(b) * d.S + seq) * d.ld_o + h * HD + (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + i * 8) = pack_bf16(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
      if ((lane & 3) == 0) lse[(static_cast<long long>(b) * d.H + h) * d.S + seq] = m_run[r] + logf(l_run[r]);
    }
  }
}

// ============================================================ backward, key-stationary -> dK, dV
// grid (ceil((nft + 1) / 2), T, B*H); consumer c owns key tile 2x + c.  Shared memory: {K, V} of each consumer, then
// LSTAGES x {Q, dO}, then LSTAGES x {lse * log2(e), delta} of the streamed query block.  A fill completes when the TMA
// bytes have landed and all 128 producer threads have written the block's lse / delta.
__global__ void __launch_bounds__(LONG_THREADS, 1)
vip_long_bwd_kv_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo,
                       const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                       const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv, float* __restrict__ gpart,
                       const AttnDims d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  float* s_stat = reinterpret_cast<float*>(sm + (4 + 2 * LSTAGES) * LTILE_BYTES);   // [LSTAGES][2][64]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(s_stat + LSTAGES * 2 * LTILE);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + LSTAGES;
  const int t = blockIdx.y, h = blockIdx.z % d.H, b = blockIdx.z / d.H;
  const int nft = num_frame_tiles(d), ntiles = nft + 1;
  const int kt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - kt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1 + 128, nlive, &tm, &tdo);
  const long long bh = static_cast<long long>(b) * d.H + h;

  if (wg == 0) {
    // ------------------------------------ producer: Q / dO by TMA, lse / delta by the whole warpgroup
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * LTILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        const int r0 = tile_row0(d, nft, b, t, kt0 + c);
        tma_load_2d(sm + 2 * c * LTILE_BYTES, &tm, q_full, d.C + h * HD, r0);
        tma_load_2d(sm + (2 * c + 1) * LTILE_BYTES, &tm, q_full, 2 * d.C + h * HD, r0);
      }
    }
    const int row = threadIdx.x >> 1, half = threadIdx.x & 1;   // two threads per query row, 32 columns each
    for (int qb = 0; qb < ntiles; ++qb) {
      const int s = qb % LSTAGES;
      mbar_wait(&empty[s], ((qb / LSTAGES) & 1) ^ 1);
      if (threadIdx.x == 0) {
        uint8_t* st = sm + (4 + 2 * s) * LTILE_BYTES;
        const int r0 = tile_row0(d, nft, b, t, qb);
        mbar_arrive_expect_tx(&full[s], 2 * LTILE_BYTES);
        tma_load_2d(st, &tm, &full[s], h * HD, r0);
        tma_load_2d(st + LTILE_BYTES, &tdo, &full[s], h * HD, r0);
      }
      const bool valid = row < tile_rows(d, nft, qb);
      float dot = 0.f;
      long long seq = 0;
      if (valid) {
        seq = tile_seq(d, nft, t, qb, row);
        const long long off = (static_cast<long long>(b) * d.S + seq) * d.ld_o + h * HD + half * 32;
        dot = dot16(dout + off, out + off) + dot16(dout + off + 16, out + off + 16);
      }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      if (half == 0) {
        s_stat[(s * 2) * LTILE + row] = valid ? lse[bh * d.S + seq] * LOG2E : INFINITY;
        s_stat[(s * 2 + 1) * LTILE + row] = dot;
      }
      mbar_arrive(&full[s]);
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, kt = kt0 + c;
  if (c >= nlive) return;
  const bool kglob = kt == nft;
  const int krows = tile_rows(d, nft, kt);
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int k_lo = wq * 16 + (lane >> 2);
  const uint32_t sK = smem_u32(sm) + 2 * c * LTILE_BYTES, sV = sK + LTILE_BYTES;
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int qb = 0; qb < ntiles; ++qb) {
    const int s = qb % LSTAGES;
    mbar_wait_nocall(&full[s], (qb / LSTAGES) & 1);
    // keys of this tile seen by the queries of block qb: the frame keys always, the global keys except for global
    // queries outside frame 0
    const int qrows = (kglob && qb == nft && t != 0) ? 0 : tile_rows(d, nft, qb);
    if (qrows == 0) {
      release_stage(empty, s);
      continue;
    }
    const uint32_t sQ = smem_u32(sm) + (4 + 2 * s) * LTILE_BYTES, sdO = sQ + LTILE_BYTES;
    const float* s_lse = s_stat + (s * 2) * LTILE;
    const float* s_delta = s_lse + LTILE;
    float st[32], dpt[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) st[i] = dpt[i] = 0.f;
    wgmma_fence_regs(st);
    wgmma_fence_regs(dpt);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      wgmma_m64n64k16_ss<0, 0>(st, kdesc(sK + ks * 32), kdesc(sQ + ks * 32));
      wgmma_m64n64k16_ss<0, 0>(dpt, kdesc(sV + ks * 32), kdesc(sdO + ks * 32));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(st);
    wgmma_fence_regs(dpt);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int q = i * 8 + (lane & 3) * 2 + (e & 1);
        const int key = k_lo + (e >> 1) * 8;
        const bool valid = q < qrows && key < krows;
        const float p = valid ? fast_exp2(fmaf(st[4 * i + e], LOG2E, -s_lse[q])) : 0.f;
        st[4 * i + e] = p;
        dpt[4 * i + e] = p * (dpt[4 * i + e] - s_delta[q]);
      }
    uint32_t ap[4][4], ad[4][4];
    acc_to_afrag(st, ap);
    acc_to_afrag(dpt, ad);
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      wgmma_m64n64k16_rs<1>(dv, ap[ks], mndesc(sdO + ks * 16 * 128));
      wgmma_m64n64k16_rs<1>(dk, ad[ks], mndesc(sQ + ks * 16 * 128));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dv);
    wgmma_fence_regs(dk);
    release_stage(empty, s);
  }
  float* gp = gpart + (bh * d.T + t) * d.M * 3 * HD;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = k_lo + r * 8;
    if (key >= krows) continue;
    if (!kglob) {
      __nv_bfloat16* row = dqkv + (static_cast<long long>(b) * d.S + tile_seq(d, nft, t, kt, key)) * d.ld_qkv + h * HD +
                           (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        *reinterpret_cast<uint32_t*>(row + d.C + i * 8) = pack_bf16(dk[4 * i + 2 * r], dk[4 * i + 2 * r + 1]);
        *reinterpret_cast<uint32_t*>(row + 2 * d.C + i * 8) = pack_bf16(dv[4 * i + 2 * r], dv[4 * i + 2 * r + 1]);
      }
    } else {
      float* g = gp + static_cast<long long>(key) * 3 * HD + (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        g[HD + i * 8] = dk[4 * i + 2 * r]; g[HD + i * 8 + 1] = dk[4 * i + 2 * r + 1];
        g[2 * HD + i * 8] = dv[4 * i + 2 * r]; g[2 * HD + i * 8 + 1] = dv[4 * i + 2 * r + 1];
      }
    }
  }
}

// ============================================================ backward, query-stationary -> dQ
// grid (ceil((nft + 1) / 2), T, B*H); consumer c owns query tile 2x + c.  Shared memory: {Q, dO} of each consumer, then
// LSTAGES x {K, V}.
__global__ void __launch_bounds__(LONG_THREADS, 1)
vip_long_bwd_q_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo,
                      const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                      const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv, float* __restrict__ gpart,
                      const AttnDims d, float q_scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (4 + 2 * LSTAGES) * LTILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + LSTAGES;
  const int t = blockIdx.y, h = blockIdx.z % d.H, b = blockIdx.z / d.H;
  const int nft = num_frame_tiles(d), ntiles = nft + 1;
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1, nlive, &tm, &tdo);
  const long long bh = static_cast<long long>(b) * d.H + h;

  if (wg == 0) {
    // ------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * LTILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        const int r0 = tile_row0(d, nft, b, t, qt0 + c);
        tma_load_2d(sm + 2 * c * LTILE_BYTES, &tm, q_full, h * HD, r0);
        tma_load_2d(sm + (2 * c + 1) * LTILE_BYTES, &tdo, q_full, h * HD, r0);
      }
      for (int kb = 0; kb < ntiles; ++kb) {
        const int s = kb % LSTAGES;
        mbar_wait_nocall(&empty[s], ((kb / LSTAGES) & 1) ^ 1);
        uint8_t* st = sm + (4 + 2 * s) * LTILE_BYTES;
        const int r0 = tile_row0(d, nft, b, t, kb);
        mbar_arrive_expect_tx(&full[s], 2 * LTILE_BYTES);
        tma_load_2d(st, &tm, &full[s], d.C + h * HD, r0);
        tma_load_2d(st + LTILE_BYTES, &tm, &full[s], 2 * d.C + h * HD, r0);
      }
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const bool qglob = qt == nft;
  const int qrows = tile_rows(d, nft, qt);
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int q_lo = wq * 16 + (lane >> 2);
  // lse * log2(e) and delta of this thread's two rows; the four lanes of a quad each sum 16 columns of delta
  float lse_r[2], del_r[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q_lo + r * 8;
    float dot = 0.f;
    lse_r[r] = INFINITY;
    if (row < qrows) {
      const long long seq = tile_seq(d, nft, t, qt, row);
      const long long off = (static_cast<long long>(b) * d.S + seq) * d.ld_o + h * HD + (lane & 3) * 16;
      dot = dot16(dout + off, out + off);
      lse_r[r] = lse[bh * d.S + seq] * LOG2E;
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    del_r[r] = dot;
  }
  const uint32_t sQ = smem_u32(sm) + 2 * c * LTILE_BYTES, sdO = sQ + LTILE_BYTES;
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % LSTAGES;
    const int klim = live_keys(d, nft, t, qt, kb);
    mbar_wait_nocall(&full[s], (kb / LSTAGES) & 1);
    if (klim == 0) {
      release_stage(empty, s);
      continue;
    }
    const uint32_t sK = smem_u32(sm) + (4 + 2 * s) * LTILE_BYTES, sV = sK + LTILE_BYTES;
    float sc[32], dp[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = dp[i] = 0.f;
    wgmma_fence_regs(sc);
    wgmma_fence_regs(dp);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      wgmma_m64n64k16_ss<0, 0>(sc, kdesc(sQ + ks * 32), kdesc(sK + ks * 32));
      wgmma_m64n64k16_ss<0, 0>(dp, kdesc(sdO + ks * 32), kdesc(sV + ks * 32));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    wgmma_fence_regs(dp);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = i * 8 + (lane & 3) * 2 + (e & 1);
        const int q = q_lo + (e >> 1) * 8;
        const bool valid = q < qrows && key < klim;
        const float p = valid ? fast_exp2(fmaf(sc[4 * i + e], LOG2E, -lse_r[e >> 1])) : 0.f;
        dp[4 * i + e] = p * (dp[4 * i + e] - del_r[e >> 1]);
      }
    uint32_t ad[4][4];
    acc_to_afrag(dp, ad);
    wgmma_fence_regs(dq);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_rs<1>(dq, ad[ks], mndesc(sK + ks * 16 * 128));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
    release_stage(empty, s);
  }
  float* gp = gpart + (bh * d.T + t) * d.M * 3 * HD;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q_lo + r * 8;
    if (q >= qrows) continue;
    if (!qglob) {
      __nv_bfloat16* row = dqkv + (static_cast<long long>(b) * d.S + tile_seq(d, nft, t, qt, q)) * d.ld_qkv + h * HD +
                           (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(row + i * 8) = pack_bf16(dq[4 * i + 2 * r] * q_scale, dq[4 * i + 2 * r + 1] * q_scale);
    } else {
      float* g = gp + static_cast<long long>(q) * 3 * HD + (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        g[i * 8] = dq[4 * i + 2 * r];
        g[i * 8 + 1] = dq[4 * i + 2 * r + 1];
      }
    }
  }
}

namespace {
constexpr int LONG_FWD_SMEM = (2 + 2 * LSTAGES) * LTILE_BYTES + 1024 + 64;
constexpr int LONG_BWD_KV_SMEM = (4 + 2 * LSTAGES) * LTILE_BYTES + LSTAGES * 2 * LTILE * 4 + 1024 + 64;
constexpr int LONG_BWD_Q_SMEM = (4 + 2 * LSTAGES) * LTILE_BYTES + 1024 + 64;

int long_grid(const AttnDims& d, dim3& grid) {
  const long long bh = static_cast<long long>(d.B) * d.H;
  if (d.T > 65535 || bh > 65535) return fail("vip_attention: T and B*H must be <= 65535");
  if (static_cast<long long>(d.B) * d.S > 0x7fffffffLL) return fail("vip_attention: B*S must fit in int32");
  const int ntiles = (d.L + LTILE - 1) / LTILE + 1;
  grid = dim3((ntiles + 1) / 2, d.T, static_cast<unsigned>(bh));
  return 0;
}
}  // namespace

int vip_long_attn_fwd(const AttnDims& d, const void* qkv, void* out, float* lse, float* part, cudaStream_t st) {
  dim3 grid;
  if (long_grid(d, grid)) return -1;
  CUtensorMap tm;
  if (make_tmap_bf16_2d(&tm, qkv, d.ld_qkv, static_cast<uint64_t>(d.B) * d.S, d.ld_qkv, HD, LTILE)) return -1;
  static bool attr = false;
  if (!attr) {
    XP_CHECK_CUDA(cudaFuncSetAttribute(vip_long_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LONG_FWD_SMEM));
    attr = true;
  }
  vip_long_fwd_kernel<<<grid, LONG_THREADS, LONG_FWD_SMEM, st>>>(tm, static_cast<__nv_bfloat16*>(out), lse, part, d);
  XP_CHECK_LAUNCH("vip_long_fwd_kernel");
  return 0;
}

int vip_long_attn_bwd(const AttnDims& d, const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                      float* gpart, float q_scale, cudaStream_t st) {
  dim3 grid;
  if (long_grid(d, grid)) return -1;
  CUtensorMap tm, tdo;
  const uint64_t rows = static_cast<uint64_t>(d.B) * d.S;
  if (make_tmap_bf16_2d(&tm, qkv, d.ld_qkv, rows, d.ld_qkv, HD, LTILE) ||
      make_tmap_bf16_2d(&tdo, dout, d.ld_o, rows, d.ld_o, HD, LTILE))
    return -1;
  static bool attr = false;
  if (!attr) {
    XP_CHECK_CUDA(
        cudaFuncSetAttribute(vip_long_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LONG_BWD_KV_SMEM));
    XP_CHECK_CUDA(
        cudaFuncSetAttribute(vip_long_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LONG_BWD_Q_SMEM));
    attr = true;
  }
  const __nv_bfloat16* o = static_cast<const __nv_bfloat16*>(out);
  const __nv_bfloat16* g = static_cast<const __nv_bfloat16*>(dout);
  __nv_bfloat16* dx = static_cast<__nv_bfloat16*>(dqkv);
  vip_long_bwd_kv_kernel<<<grid, LONG_THREADS, LONG_BWD_KV_SMEM, st>>>(tm, tdo, o, g, lse, dx, gpart, d);
  XP_CHECK_LAUNCH("vip_long_bwd_kv_kernel");
  vip_long_bwd_q_kernel<<<grid, LONG_THREADS, LONG_BWD_Q_SMEM, st>>>(tm, tdo, o, g, lse, dx, gpart, d, q_scale);
  XP_CHECK_LAUNCH("vip_long_bwd_q_kernel");
  return 0;
}

}  // namespace xp
