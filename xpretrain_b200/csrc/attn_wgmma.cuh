// The wgmma attention core (head_dim 64, bf16 operands, fp32 accumulators) shared by the staged proxy-token kernels
// (vip_attention.cu), the streamed proxy-token kernels (vip_attention_long.cu) and the dense kernels (dense_attention.cu).
//
// Per-block steps.  One warpgroup owns a 64-row tile and meets one 64-row block of the other side per step; every product
// is a wgmma with both operands in 128B-swizzled shared memory, or P / dS as the register A operand.  Element 4 i + e of a
// 64 x 64 accumulator sits in tile-local row wq * 16 + lane / 4 + 8 (e >> 1) and column 8 i + 2 (lane & 3) + (e & 1).
//   fwd_step   S = Q·Kᵀ, online softmax in registers, O += P·V with P split into bf16 hi + lo (P = hi + lo to ~2^-16:
//              rounding P to bf16 is the largest error of the forward, and it reaches the pooled CLS features);
//   kv_step    Sᵀ = K·Qᵀ and dPᵀ = V·dOᵀ, then dV += Pᵀ·dO and dK += dSᵀ·Q (key-stationary);
//   q_step     S = Q·Kᵀ and dP = dO·Vᵀ, then dQ += dS·K (query-stationary).
// No operand is transposed in memory: V, dO, Q and K serve as MN-major B operands where a product contracts over their
// rows.  Each step takes a predicate live(q, key) over tile-local query and key indices; dead pairs get a -inf logit
// (forward) or P = 0 (backward).
//
// Streamed pipeline (stream_*_kernel), FlashAttention-3 shaped, for sequences too long to stage whole: a CTA of three
// warpgroups per two 64-row tiles.  Warpgroup 0 is the producer (setmaxnreg down to 40): one thread streams 64-row blocks
// by TMA into shared memory through a STAGES-deep full / empty mbarrier ring.  Warpgroups 1 and 2 are consumers
// (setmaxnreg up to 232), each owning one tile:
//   forward    query-stationary, K / V blocks streamed, fwd_step per block;
//   backward   key-stationary kernel: Q / dO blocks streamed, kv_step per block; the producer warpgroup also writes each
//              block's lse * log2(e) and delta = rowsum(dO * O) into the stage;
//              query-stationary kernel: K / V blocks streamed, q_step per block.
// A layout policy P says where the tiles of a CTA lie and what its epilogues store:
//   STAGES                     ring depth;
//   bind()                     derive the CTA's coordinates from blockIdx once, on the kernel's local copy of the
//                              policy (the compiler does not hoist a division out of loops that wait on barriers);
//   ntiles()                   64-row tiles of the CTA's sequence (grid.x = ceil(ntiles / 2));
//   load(dst, tm, bar, m, j)   TMA of column block m (0: Q or dO, 1: K, 2: V) of tile j;
//   rows(j)                    live rows of tile j, a prefix of the tile (>= 1);
//   skip(qt, kt)               query tile qt and key tile kt share no live pair: the block is passed over;
//   ZERO_FILL                  rows past a tile's live rows load as zeros, so the backward kernels need no row mask:
//                              such a query row has P = 0 exactly (zero Q and dO, lse = +inf), and such a key row
//                              only feeds dK / dV rows that are never stored.  Otherwise they may hold any value,
//                              NaN included, and are masked;
//   fill_stats(s, qb)          all 128 producer threads: s[0, 64) = lse * log2(e) (+inf past the live rows, so that
//                              P = 0 there), s[64, 128) = delta of query block qb;
//   row_stats(qt, q_lo, l, d)  every consumer lane: lse * log2(e) and delta of rows q_lo and q_lo + 8 of query tile qt;
//   store_fwd / store_kv / store_q   one live row of an epilogue.
// Every output element has exactly one writer and no float atomics are used, so results do not depend on scheduling.
#pragma once
#include "ptx.cuh"
#include "mma_frag.cuh"

namespace xp {

constexpr int ATILE = 64;                  // rows per tile / streamed block
constexpr int ATILE_BYTES = ATILE * 128;   // one [64][64] bf16 tile, 128B-swizzled
constexpr int STREAM_THREADS = 384;        // producer warpgroup + two consumer warpgroups

// Dynamic shared memory of the streamed kernels: two consumers' own tiles, the ring, the kv kernel's per-stage
// {lse, delta}, then the barriers, plus the slack of aligning the base to 1024 bytes.
constexpr int stream_fwd_smem(int stages) { return (2 + 2 * stages) * ATILE_BYTES + 1024 + 64; }
constexpr int stream_kv_smem(int stages) { return (4 + 2 * stages) * ATILE_BYTES + stages * 2 * ATILE * 4 + 1024 + 64; }
constexpr int stream_q_smem(int stages) { return (4 + 2 * stages) * ATILE_BYTES + 1024 + 64; }

__device__ __forceinline__ uint64_t kdesc(uint32_t addr) { return make_smem_desc_sw128(addr, 16, 1024); }     // K-major
__device__ __forceinline__ uint64_t mndesc(uint32_t addr) { return make_smem_desc_sw128(addr, 8192, 1024); }  // MN-major

// P (or dS) of a 64 x 64 accumulator as the A fragments of the four k16 steps: k-step ks covers columns [16 ks, 16 ks + 16)
__device__ __forceinline__ void acc_to_afrag(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16(x[8 * ks + 0], x[8 * ks + 1]);
    a[ks][1] = pack_bf16(x[8 * ks + 2], x[8 * ks + 3]);
    a[ks][2] = pack_bf16(x[8 * ks + 4], x[8 * ks + 5]);
    a[ks][3] = pack_bf16(x[8 * ks + 6], x[8 * ks + 7]);
  }
}

// ------------------------------------------------------------------------------------------- per-block steps
// partial = false: every pair of the block is live, and the predicate is not evaluated
template <class Live>
__device__ __forceinline__ void fwd_step(uint32_t sQ, uint32_t sK, uint32_t sV, float (&o)[32], float (&m_run)[2],
                                         float (&l_run)[2], Live live, bool partial = true) {
  const int lane = threadIdx.x & 31, q_lo = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  float s[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) s[i] = 0.f;
  wgmma_fence_regs(s);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_ss<0, 0>(s, kdesc(sQ + ks * 32), kdesc(sK + ks * 32));
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  if (partial) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (!live(q_lo + (e >> 1) * 8, i * 8 + (lane & 3) * 2 + (e & 1))) s[4 * i + e] = -INFINITY;
  }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 32; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
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
    const float pv = fast_exp2(fmaf(s[i], LOG2E, -mb[(i >> 1) & 1]));   // exp2(-inf) = 0 for masked entries
    s[i] = pv;
    l_run[(i >> 1) & 1] += pv;
  }
  uint32_t ph[4][4], pl[4][4];
  acc_to_afrag(s, ph);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      pl[ks][j] = pack_bf16(s[8 * ks + 2 * j] - bf16_lo(ph[ks][j]), s[8 * ks + 2 * j + 1] - bf16_hi(ph[ks][j]));
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
}

// l_run of fwd_step holds each lane's share of its rows' sums; add the four lanes of the quad
__device__ __forceinline__ void quad_sum(float (&l_run)[2]) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
}

// s_lse / s_delta: lse * log2(e) and delta of the block's 64 query rows
template <class Live>
__device__ __forceinline__ void kv_step(uint32_t sK, uint32_t sV, uint32_t sQ, uint32_t sdO, const float* s_lse,
                                        const float* s_delta, float (&dk)[32], float (&dv)[32], Live live) {
  const int lane = threadIdx.x & 31, k_lo = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
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
      const float p = live(q, k_lo + (e >> 1) * 8) ? fast_exp2(fmaf(st[4 * i + e], LOG2E, -s_lse[q])) : 0.f;
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
}

// lse_r / del_r: lse * log2(e) and delta of this thread's rows q_lo and q_lo + 8
template <class Live>
__device__ __forceinline__ void q_step(uint32_t sQ, uint32_t sdO, uint32_t sK, uint32_t sV, const float (&lse_r)[2],
                                       const float (&del_r)[2], float (&dq)[32], Live live) {
  const int lane = threadIdx.x & 31, q_lo = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  float s[32], dp[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) s[i] = dp[i] = 0.f;
  wgmma_fence_regs(s);
  wgmma_fence_regs(dp);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    wgmma_m64n64k16_ss<0, 0>(s, kdesc(sQ + ks * 32), kdesc(sK + ks * 32));
    wgmma_m64n64k16_ss<0, 0>(dp, kdesc(sdO + ks * 32), kdesc(sV + ks * 32));
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(s);
  wgmma_fence_regs(dp);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const bool valid = live(q_lo + (e >> 1) * 8, i * 8 + (lane & 3) * 2 + (e & 1));
      const float p = valid ? fast_exp2(fmaf(s[4 * i + e], LOG2E, -lse_r[e >> 1])) : 0.f;
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
}

// ----------------------------------------------------------------------------------------- streamed pipeline
// Barrier set-up of the ring; `full_count` arrivals complete a fill, every live consumer warp releases a stage.
template <int STAGES>
__device__ __forceinline__ void init_ring(uint64_t* q_full, uint64_t* full, uint64_t* empty, uint32_t full_count,
                                          int nlive, const CUtensorMap* tm0, const CUtensorMap* tm1) {
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tm0);
    tma_prefetch_desc(tm1);
    mbar_init(q_full, 1);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
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

// One thread: stream K / V of every tile through the ring at tile offset `ring` of the shared memory.
template <class P>
__device__ __forceinline__ void produce_kv_blocks(const P& p, const CUtensorMap* tm, uint8_t* sm, int ring,
                                                  uint64_t* full, uint64_t* empty) {
  for (int kb = 0; kb < p.ntiles(); ++kb) {
    const int s = kb % P::STAGES;
    mbar_wait_nocall(&empty[s], ((kb / P::STAGES) & 1) ^ 1);
    uint8_t* st = sm + (ring + 2 * s) * ATILE_BYTES;
    mbar_arrive_expect_tx(&full[s], 2 * ATILE_BYTES);
    p.load(st, tm, &full[s], 1, kb);
    p.load(st + ATILE_BYTES, tm, &full[s], 2, kb);
  }
}

// Each kernel rounds its dynamic shared memory up to 1024 bytes in place: behind a helper function, ptxas loses the
// alignment and no longer pairs the per-row lse / delta loads of kv_step.
//
// forward: grid (ceil(ntiles / 2), ...); consumer c of CTA x owns query tile 2x + c.  Shared memory: the two Q tiles,
// then STAGES x {K, V}.
template <class P>
__global__ void __launch_bounds__(STREAM_THREADS, 1)
stream_fwd_kernel(const __grid_constant__ CUtensorMap tm, const P layout) {
  P p = layout;
  p.bind();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (2 + 2 * P::STAGES) * ATILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + P::STAGES;
  const int ntiles = p.ntiles();
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring<P::STAGES>(q_full, full, empty, 1, nlive, &tm, &tm);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * ATILE_BYTES);
      for (int c = 0; c < nlive; ++c) p.load(sm + c * ATILE_BYTES, &tm, q_full, 0, qt0 + c);
      produce_kv_blocks(p, &tm, sm, 2, full, empty);
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const int r_lo = ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2);
  const uint32_t sQ = smem_u32(sm) + c * ATILE_BYTES;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % P::STAGES;
    const int klim = p.skip(qt, kb) ? 0 : p.rows(kb);   // live keys of the block, 0: pass it over
    mbar_wait_nocall(&full[s], (kb / P::STAGES) & 1);
    if (klim != 0) {
      const uint32_t sK = smem_u32(sm) + (2 + 2 * s) * ATILE_BYTES;
      fwd_step(sQ, sK, sK + ATILE_BYTES, o, m_run, l_run, [&](int, int key) { return key < klim; }, klim < ATILE);
    }
    release_stage(empty, s);
  }
  quad_sum(l_run);
  const int qrows = p.rows(qt);
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (r_lo + r * 8 < qrows) p.store_fwd(qt, r_lo + r * 8, r, o, m_run[r], l_run[r]);
}

// backward, key-stationary -> dK, dV: consumer c owns key tile 2x + c.  Shared memory: {K, V} of each consumer, then
// STAGES x {Q, dO}, then STAGES x {lse * log2(e), delta}.  A fill completes when the TMA bytes have landed and all 128
// producer threads have written the block's lse / delta.
template <class P>
__global__ void __launch_bounds__(STREAM_THREADS, 1)
stream_bwd_kv_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo, const P layout) {
  P p = layout;
  p.bind();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  float* s_stat = reinterpret_cast<float*>(sm + (4 + 2 * P::STAGES) * ATILE_BYTES);   // [STAGES][2][64]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(s_stat + P::STAGES * 2 * ATILE);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + P::STAGES;
  const int ntiles = p.ntiles();
  const int kt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - kt0);
  const int wg = threadIdx.x >> 7;
  init_ring<P::STAGES>(q_full, full, empty, 1 + 128, nlive, &tm, &tdo);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * ATILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        p.load(sm + 2 * c * ATILE_BYTES, &tm, q_full, 1, kt0 + c);
        p.load(sm + (2 * c + 1) * ATILE_BYTES, &tm, q_full, 2, kt0 + c);
      }
    }
    for (int qb = 0; qb < ntiles; ++qb) {
      const int s = qb % P::STAGES;
      mbar_wait(&empty[s], ((qb / P::STAGES) & 1) ^ 1);
      if (threadIdx.x == 0) {
        uint8_t* st = sm + (4 + 2 * s) * ATILE_BYTES;
        mbar_arrive_expect_tx(&full[s], 2 * ATILE_BYTES);
        p.load(st, &tm, &full[s], 0, qb);
        p.load(st + ATILE_BYTES, &tdo, &full[s], 0, qb);
      }
      p.fill_stats(s_stat + s * 2 * ATILE, qb);
      mbar_arrive(&full[s]);
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1, kt = kt0 + c;
  if (c >= nlive) return;
  const int krows = p.rows(kt);
  const int k_lo = ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2);
  const uint32_t sK = smem_u32(sm) + 2 * c * ATILE_BYTES;
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int qb = 0; qb < ntiles; ++qb) {
    const int s = qb % P::STAGES;
    mbar_wait_nocall(&full[s], (qb / P::STAGES) & 1);
    if (!p.skip(qb, kt)) {
      const int qrows = p.rows(qb);
      const uint32_t sQ = smem_u32(sm) + (4 + 2 * s) * ATILE_BYTES;
      const float* s_lse = s_stat + s * 2 * ATILE;
      kv_step(sK, sK + ATILE_BYTES, sQ, sQ + ATILE_BYTES, s_lse, s_lse + ATILE, dk, dv,
              [&](int q, int key) { return P::ZERO_FILL || (q < qrows && key < krows); });
    }
    release_stage(empty, s);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (k_lo + r * 8 < krows) p.store_kv(kt, k_lo + r * 8, r, dk, dv);
}

// backward, query-stationary -> dQ: consumer c owns query tile 2x + c.  Shared memory: {Q, dO} of each consumer, then
// STAGES x {K, V}.
template <class P>
__global__ void __launch_bounds__(STREAM_THREADS, 1)
stream_bwd_q_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo, const P layout) {
  P p = layout;
  p.bind();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (4 + 2 * P::STAGES) * ATILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + P::STAGES;
  const int ntiles = p.ntiles();
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring<P::STAGES>(q_full, full, empty, 1, nlive, &tm, &tdo);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * ATILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        p.load(sm + 2 * c * ATILE_BYTES, &tm, q_full, 0, qt0 + c);
        p.load(sm + (2 * c + 1) * ATILE_BYTES, &tdo, q_full, 0, qt0 + c);
      }
      produce_kv_blocks(p, &tm, sm, 4, full, empty);
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const int qrows = p.rows(qt);
  const int q_lo = ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2);
  float lse_r[2], del_r[2];
  p.row_stats(qt, q_lo, lse_r, del_r);
  const uint32_t sQ = smem_u32(sm) + 2 * c * ATILE_BYTES;
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % P::STAGES;
    const bool live = !p.skip(qt, kb);
    const int klim = p.rows(kb);
    mbar_wait_nocall(&full[s], (kb / P::STAGES) & 1);
    if (live) {
      const uint32_t sK = smem_u32(sm) + (4 + 2 * s) * ATILE_BYTES;
      q_step(sQ, sQ + ATILE_BYTES, sK, sK + ATILE_BYTES, lse_r, del_r, dq,
             [&](int q, int key) { return (P::ZERO_FILL || q < qrows) && key < klim; });
    }
    release_stage(empty, s);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r)
    if (q_lo + r * 8 < qrows) p.store_q(qt, q_lo + r * 8, r, dq);
}

}  // namespace xp
