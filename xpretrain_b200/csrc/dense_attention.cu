// Dense (non-causal, unmasked) multi-head attention, head_dim 64, over sequences of consecutive rows of the fused
// token-major qkv buffer: the joint space-time and space-only attentions of HD-VILA's TimeSformer (Attention.forward,
// timesformer.py:156-173, on x of shape [B, H*W*T, C] or [B*T, H*W, C], :202-205).  See xp_dense_attention_* in
// include/xpretrain_b200.h for the ABI.
//
// Hopper path, FlashAttention-3 shaped, like vip_attention_long.cu: a CTA of three warpgroups per two 64-row tiles of
// one (sequence, head).  Warpgroup 0 is the producer (setmaxnreg down to 40): one thread streams 64-row blocks by TMA
// into 128B-swizzled shared memory through an LSTAGES-deep full / empty mbarrier ring.  Warpgroups 1 and 2 are consumers
// (setmaxnreg up to 232), each owning one tile, with every product on wgmma:
//   forward    query-stationary: S = Q·Kᵀ, online softmax over the 64-key blocks in registers, O += P·V with P in
//              registers, split into bf16 hi + lo (rounding P is the largest error of a plain bf16 P·V);
//   backward   delta = rowsum(dO * O) by a small kernel, then
//              key-stationary kernel: Sᵀ = K·Qᵀ and dPᵀ = V·dOᵀ per streamed query block, dV += Pᵀ·dO, dK += dSᵀ·Q;
//              the producer warpgroup also loads each block's LSE and delta;
//              query-stationary kernel: S = Q·Kᵀ and dP = dO·Vᵀ per streamed key block, dQ += dS·K.
//
// Sequences are ragged against the 64-row tiles (392, 1120 and 6272 rows are not multiples of 64), and the next sequence
// sits directly behind the last one.  Every tile is loaded through a 3-D tensor map {columns, seq_len, n_seq}: box rows
// past the end of the sequence are zero-filled by the TMA unit, so no value of a neighbouring sequence (not even a NaN)
// reaches the products.  Keys past the end get a -inf logit (forward) or P = 0 (dQ); query rows past the end have zero Q
// and dO and an LSE of +inf, so that their P is exactly 0 in the key-stationary kernel; they are never written.
// Every output element has exactly one writer and no float atomics are used, so results do not depend on scheduling.
#include <algorithm>

#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"
#include "mma_frag.cuh"

namespace xp {

namespace {

constexpr int DTILE = 64;                   // rows per tile / streamed block
constexpr int DTILE_BYTES = DTILE * 128;    // one [64][64] bf16 tile, 128B-swizzled
constexpr int DENSE_THREADS = 384;          // producer warpgroup + two consumer warpgroups
constexpr int DSTAGES = 3;                  // ring depth of the streamed blocks

struct DenseDims {
  long long n_rows, ld_qkv, ld_o;
  int H, n_seq, L, C;
};

__device__ __forceinline__ uint64_t kdesc(uint32_t addr) { return make_smem_desc_sw128(addr, 16, 1024); }     // K-major
__device__ __forceinline__ uint64_t mndesc(uint32_t addr) { return make_smem_desc_sw128(addr, 8192, 1024); }  // MN-major

__device__ __forceinline__ int num_tiles(const DenseDims& d) { return (d.L + DTILE - 1) / DTILE; }
__device__ __forceinline__ int live_rows(const DenseDims& d, int j) { return min(DTILE, d.L - j * DTILE); }

__device__ __forceinline__ void acc_to_afrag(const float (&x)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16(x[8 * ks + 0], x[8 * ks + 1]);
    a[ks][1] = pack_bf16(x[8 * ks + 2], x[8 * ks + 3]);
    a[ks][2] = pack_bf16(x[8 * ks + 4], x[8 * ks + 5]);
    a[ks][3] = pack_bf16(x[8 * ks + 6], x[8 * ks + 7]);
  }
}

// Barrier set-up of the ring; `full_count` arrivals complete a fill, every live consumer warp releases a stage.
__device__ __forceinline__ void init_ring(uint64_t* q_full, uint64_t* full, uint64_t* empty, uint32_t full_count,
                                          int nlive, const CUtensorMap* tm0, const CUtensorMap* tm1) {
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tm0);
    tma_prefetch_desc(tm1);
    mbar_init(q_full, 1);
#pragma unroll
    for (int s = 0; s < DSTAGES; ++s) {
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
// grid (ceil(ntiles / 2), H, n_seq); consumer c of CTA x owns query tile 2x + c.  Shared memory: the two Q tiles, then
// DSTAGES x {K, V}.
__global__ void __launch_bounds__(DENSE_THREADS, 1)
dense_fwd_kernel(const __grid_constant__ CUtensorMap tm, __nv_bfloat16* __restrict__ out, float* __restrict__ lse,
                 const DenseDims d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (2 + 2 * DSTAGES) * DTILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + DSTAGES;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int ntiles = num_tiles(d);
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1, nlive, &tm, &tm);

  if (wg == 0) {
    // ------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * DTILE_BYTES);
      for (int c = 0; c < nlive; ++c) tma_load_3d(sm + c * DTILE_BYTES, &tm, q_full, h * HD, (qt0 + c) * DTILE, seq);
      for (int kb = 0; kb < ntiles; ++kb) {
        const int s = kb % DSTAGES;
        mbar_wait_nocall(&empty[s], ((kb / DSTAGES) & 1) ^ 1);
        uint8_t* st = sm + (2 + 2 * s) * DTILE_BYTES;
        mbar_arrive_expect_tx(&full[s], 2 * DTILE_BYTES);
        tma_load_3d(st, &tm, &full[s], d.C + h * HD, kb * DTILE, seq);
        tma_load_3d(st + DTILE_BYTES, &tm, &full[s], 2 * d.C + h * HD, kb * DTILE, seq);
      }
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int r_lo = wq * 16 + (lane >> 2);
  const uint32_t sQ = smem_u32(sm) + c * DTILE_BYTES;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % DSTAGES;
    const int klim = live_rows(d, kb);
    mbar_wait_nocall(&full[s], (kb / DSTAGES) & 1);
    const uint32_t sK = smem_u32(sm) + (2 + 2 * s) * DTILE_BYTES, sV = sK + DTILE_BYTES;
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
    if (klim < DTILE) {   // the last block of a ragged sequence: keys past the end (zero-filled rows) get no weight
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (i * 8 + (lane & 3) * 2 + (e & 1) >= klim) sc[4 * i + e] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
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
    // P·V with P = hi + lo in bf16
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
  const int qrows = live_rows(d, qt);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r_lo + r * 8;
    if (row >= qrows) continue;
    const long long grow = static_cast<long long>(seq) * d.L + qt * DTILE + row;
    const float inv = 1.f / l_run[r];   // > 0: every query sees at least one key
    __nv_bfloat16* dst = out + grow * d.ld_o + h * HD + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + i * 8) = pack_bf16(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
    if ((lane & 3) == 0) lse[static_cast<long long>(h) * d.n_rows + grow] = m_run[r] + logf(l_run[r]);
  }
}

// ============================================================ backward: delta = rowsum(dO * O)
// Eight threads per (row, head), 8 columns each, summed in a fixed shuffle order.  grid-stride over n_seq * L * H rows.
// The item count is a multiple of 8, so the eight lanes of a group are always active together.
__global__ void __launch_bounds__(256)
dense_delta_kernel(const __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ dout,
                   float* __restrict__ delta, const DenseDims d) {
  const long long rows = static_cast<long long>(d.n_seq) * d.L;
  const long long items = rows * d.H * 8;
  const unsigned group = 0xffu << (threadIdx.x & 24);
  for (long long it = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; it < items;
       it += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int part = static_cast<int>(it & 7);
    const long long rh = it >> 3;
    const long long row = rh / d.H;
    const int h = static_cast<int>(rh - row * d.H);
    const long long off = row * d.ld_o + h * HD + part * 8;
    const uint4 gv = *reinterpret_cast<const uint4*>(dout + off), ov = *reinterpret_cast<const uint4*>(out + off);
    const uint32_t gw[4] = {gv.x, gv.y, gv.z, gv.w}, ow[4] = {ov.x, ov.y, ov.z, ov.w};
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) acc += bf16_lo(gw[i]) * bf16_lo(ow[i]) + bf16_hi(gw[i]) * bf16_hi(ow[i]);
    acc += __shfl_xor_sync(group, acc, 1);
    acc += __shfl_xor_sync(group, acc, 2);
    acc += __shfl_xor_sync(group, acc, 4);
    if (part == 0) delta[static_cast<long long>(h) * d.n_rows + row] = acc;
  }
}

// ============================================================ backward, key-stationary -> dK, dV
// grid (ceil(ntiles / 2), H, n_seq); consumer c owns key tile 2x + c.  Shared memory: {K, V} of each consumer, then
// DSTAGES x {Q, dO}, then DSTAGES x {lse * log2(e), delta} of the streamed query block.  A fill completes when the TMA
// bytes have landed and all 128 producer threads have written the block's lse / delta.
__global__ void __launch_bounds__(DENSE_THREADS, 1)
dense_bwd_kv_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo,
                    const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                    const DenseDims d) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  float* s_stat = reinterpret_cast<float*>(sm + (4 + 2 * DSTAGES) * DTILE_BYTES);   // [DSTAGES][2][64]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(s_stat + DSTAGES * 2 * DTILE);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + DSTAGES;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int ntiles = num_tiles(d);
  const int kt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - kt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1 + 128, nlive, &tm, &tdo);
  const long long row0 = static_cast<long long>(seq) * d.L;   // first row of the sequence

  if (wg == 0) {
    // ------------------------------------ producer: Q / dO by TMA, lse / delta by the whole warpgroup
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * DTILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        tma_load_3d(sm + 2 * c * DTILE_BYTES, &tm, q_full, d.C + h * HD, (kt0 + c) * DTILE, seq);
        tma_load_3d(sm + (2 * c + 1) * DTILE_BYTES, &tm, q_full, 2 * d.C + h * HD, (kt0 + c) * DTILE, seq);
      }
    }
    const int row = threadIdx.x & 63, which = threadIdx.x >> 6;   // threads 0-63: lse, 64-127: delta
    const float* src = (which == 0 ? lse : delta) + static_cast<long long>(h) * d.n_rows + row0;
    for (int qb = 0; qb < ntiles; ++qb) {
      const int s = qb % DSTAGES;
      mbar_wait(&empty[s], ((qb / DSTAGES) & 1) ^ 1);
      if (threadIdx.x == 0) {
        uint8_t* st = sm + (4 + 2 * s) * DTILE_BYTES;
        mbar_arrive_expect_tx(&full[s], 2 * DTILE_BYTES);
        tma_load_3d(st, &tm, &full[s], h * HD, qb * DTILE, seq);
        tma_load_3d(st + DTILE_BYTES, &tdo, &full[s], h * HD, qb * DTILE, seq);
      }
      const bool valid = row < live_rows(d, qb);
      // rows past the end: lse = +inf gives P = 0 exactly (their Q and dO are zero-filled, so every product is finite)
      const float v = valid ? src[qb * DTILE + row] : 0.f;
      s_stat[(s * 2 + which) * DTILE + row] = which == 0 ? (valid ? v * LOG2E : INFINITY) : v;
      mbar_arrive(&full[s]);
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, kt = kt0 + c;
  if (c >= nlive) return;
  const int krows = live_rows(d, kt);
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int k_lo = wq * 16 + (lane >> 2);
  const uint32_t sK = smem_u32(sm) + 2 * c * DTILE_BYTES, sV = sK + DTILE_BYTES;
  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int qb = 0; qb < ntiles; ++qb) {
    const int s = qb % DSTAGES;
    mbar_wait_nocall(&full[s], (qb / DSTAGES) & 1);
    const uint32_t sQ = smem_u32(sm) + (4 + 2 * s) * DTILE_BYTES, sdO = sQ + DTILE_BYTES;
    const float* s_lse = s_stat + (s * 2) * DTILE;
    const float* s_delta = s_lse + DTILE;
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
        const float p = fast_exp2(fmaf(st[4 * i + e], LOG2E, -s_lse[q]));
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
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = k_lo + r * 8;
    if (key >= krows) continue;
    __nv_bfloat16* row = dqkv + (row0 + kt * DTILE + key) * d.ld_qkv + h * HD + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      *reinterpret_cast<uint32_t*>(row + d.C + i * 8) = pack_bf16(dk[4 * i + 2 * r], dk[4 * i + 2 * r + 1]);
      *reinterpret_cast<uint32_t*>(row + 2 * d.C + i * 8) = pack_bf16(dv[4 * i + 2 * r], dv[4 * i + 2 * r + 1]);
    }
  }
}

// ============================================================ backward, query-stationary -> dQ
// grid (ceil(ntiles / 2), H, n_seq); consumer c owns query tile 2x + c.  Shared memory: {Q, dO} of each consumer, then
// DSTAGES x {K, V}.
__global__ void __launch_bounds__(DENSE_THREADS, 1)
dense_bwd_q_kernel(const __grid_constant__ CUtensorMap tm, const __grid_constant__ CUtensorMap tdo,
                   const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                   const DenseDims d, float q_scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + (((smem_u32(smem_raw) + 1023u) & ~1023u) - smem_u32(smem_raw));
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sm + (4 + 2 * DSTAGES) * DTILE_BYTES);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + DSTAGES;
  const int h = blockIdx.y, seq = blockIdx.z;
  const int ntiles = num_tiles(d);
  const int qt0 = 2 * blockIdx.x;
  const int nlive = min(2, ntiles - qt0);
  const int wg = threadIdx.x >> 7;
  init_ring(q_full, full, empty, 1, nlive, &tm, &tdo);
  const long long row0 = static_cast<long long>(seq) * d.L;

  if (wg == 0) {
    // ------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(q_full, nlive * 2 * DTILE_BYTES);
      for (int c = 0; c < nlive; ++c) {
        tma_load_3d(sm + 2 * c * DTILE_BYTES, &tm, q_full, h * HD, (qt0 + c) * DTILE, seq);
        tma_load_3d(sm + (2 * c + 1) * DTILE_BYTES, &tdo, q_full, h * HD, (qt0 + c) * DTILE, seq);
      }
      for (int kb = 0; kb < ntiles; ++kb) {
        const int s = kb % DSTAGES;
        mbar_wait_nocall(&empty[s], ((kb / DSTAGES) & 1) ^ 1);
        uint8_t* st = sm + (4 + 2 * s) * DTILE_BYTES;
        mbar_arrive_expect_tx(&full[s], 2 * DTILE_BYTES);
        tma_load_3d(st, &tm, &full[s], d.C + h * HD, kb * DTILE, seq);
        tma_load_3d(st + DTILE_BYTES, &tm, &full[s], 2 * d.C + h * HD, kb * DTILE, seq);
      }
    }
    return;
  }
  // -------------------------------------------------------- consumers
  setmaxnreg_inc<232>();
  const int c = wg - 1, qt = qt0 + c;
  if (c >= nlive) return;
  const int qrows = live_rows(d, qt);
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int q_lo = wq * 16 + (lane >> 2);
  // lse * log2(e) and delta of this thread's two rows (+inf / 0 past the end: P = 0)
  float lse_r[2], del_r[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = q_lo + r * 8;
    const long long at = static_cast<long long>(h) * d.n_rows + row0 + qt * DTILE + row;
    lse_r[r] = row < qrows ? lse[at] * LOG2E : INFINITY;
    del_r[r] = row < qrows ? delta[at] : 0.f;
  }
  const uint32_t sQ = smem_u32(sm) + 2 * c * DTILE_BYTES, sdO = sQ + DTILE_BYTES;
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait_nocall(q_full, 0);
#pragma unroll 1
  for (int kb = 0; kb < ntiles; ++kb) {
    const int s = kb % DSTAGES;
    const int klim = live_rows(d, kb);
    mbar_wait_nocall(&full[s], (kb / DSTAGES) & 1);
    const uint32_t sK = smem_u32(sm) + (4 + 2 * s) * DTILE_BYTES, sV = sK + DTILE_BYTES;
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
        const float p = key < klim ? fast_exp2(fmaf(sc[4 * i + e], LOG2E, -lse_r[e >> 1])) : 0.f;
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
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q_lo + r * 8;
    if (q >= qrows) continue;
    __nv_bfloat16* row = dqkv + (row0 + qt * DTILE + q) * d.ld_qkv + h * HD + (lane & 3) * 2;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(row + i * 8) = pack_bf16(dq[4 * i + 2 * r] * q_scale, dq[4 * i + 2 * r + 1] * q_scale);
  }
}

namespace {
constexpr int DENSE_FWD_SMEM = (2 + 2 * DSTAGES) * DTILE_BYTES + 1024 + 64;
constexpr int DENSE_BWD_KV_SMEM = (4 + 2 * DSTAGES) * DTILE_BYTES + DSTAGES * 2 * DTILE * 4 + 1024 + 64;
constexpr int DENSE_BWD_Q_SMEM = (4 + 2 * DSTAGES) * DTILE_BYTES + 1024 + 64;

int to_dims(const XpDenseAttn* a, DenseDims& d, const char* who) {
  if (a == nullptr) return fail(std::string(who) + ": null descriptor");
  if (a->heads <= 0 || a->n_seq <= 0 || a->seq_len <= 0) return fail(std::string(who) + ": heads, n_seq, seq_len >= 1");
  if (a->n_seq > 65535 || a->heads > 65535) return fail(std::string(who) + ": n_seq and heads must be <= 65535");
  const long long rows = static_cast<long long>(a->n_seq) * a->seq_len;
  if (a->n_rows < rows) return fail(std::string(who) + ": n_rows < n_seq * seq_len");
  if (a->n_rows * a->heads >= (1LL << 31) || a->n_rows >= (1LL << 31))
    return fail(std::string(who) + ": heads * n_rows must be < 2^31");
  const long long C = 64LL * a->heads;
  if (a->ld_qkv < 3 * C || a->ld_out < C || a->ld_qkv % 8 || a->ld_out % 8)
    return fail(std::string(who) + ": ld_qkv >= 3*heads*64, ld_out >= heads*64, both multiples of 8");
  d.n_rows = a->n_rows;
  d.ld_qkv = a->ld_qkv;
  d.ld_o = a->ld_out;
  d.H = a->heads;
  d.n_seq = a->n_seq;
  d.L = a->seq_len;
  d.C = static_cast<int>(C);
  return 0;
}

dim3 dense_grid(const DenseDims& d) {
  const int ntiles = (d.L + DTILE - 1) / DTILE;
  return dim3((ntiles + 1) / 2, d.H, d.n_seq);
}

// {columns, seq_len, n_seq} view of a token-major [rows, ld] buffer: box rows past a sequence's end read as zero
int seq_tmap(CUtensorMap* tm, const void* base, long long ld, const DenseDims& d) {
  return make_tmap_bf16_3d(tm, base, ld, d.L, d.n_seq, ld, ld * d.L, HD, DTILE);
}
}  // namespace

}  // namespace xp

using namespace xp;

extern "C" int xp_dense_attention_fwd(const void* qkv, void* out, float* lse, const XpDenseAttn* desc, void* stream) {
  XP_ENTER(qkv);
  DenseDims d;
  if (int rc = to_dims(desc, d, "xp_dense_attention_fwd")) return rc;
  CUtensorMap tm;
  if (seq_tmap(&tm, qkv, d.ld_qkv, d)) return -1;
  static bool attr = false;
  if (!attr) {
    XP_CHECK_CUDA(cudaFuncSetAttribute(dense_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DENSE_FWD_SMEM));
    attr = true;
  }
  dense_fwd_kernel<<<dense_grid(d), DENSE_THREADS, DENSE_FWD_SMEM, static_cast<cudaStream_t>(stream)>>>(
      tm, static_cast<__nv_bfloat16*>(out), lse, d);
  XP_CHECK_LAUNCH("dense_fwd_kernel");
  return 0;
}

extern "C" int xp_dense_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                                      void* dqkv, const XpDenseAttn* desc, float q_scale, void* stream) {
  XP_ENTER(qkv);
  DenseDims d;
  if (int rc = to_dims(desc, d, "xp_dense_attention_bwd")) return rc;
  if ((reinterpret_cast<uintptr_t>(out) & 15) != 0) return fail("xp_dense_attention_bwd: out must be 16-byte aligned");
  CUtensorMap tm, tdo;
  if (seq_tmap(&tm, qkv, d.ld_qkv, d) || seq_tmap(&tdo, dout, d.ld_o, d)) return -1;
  static bool attr = false;
  if (!attr) {
    XP_CHECK_CUDA(
        cudaFuncSetAttribute(dense_bwd_kv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DENSE_BWD_KV_SMEM));
    XP_CHECK_CUDA(cudaFuncSetAttribute(dense_bwd_q_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DENSE_BWD_Q_SMEM));
    attr = true;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long items = static_cast<long long>(d.n_seq) * d.L * d.H * 8;
  const unsigned blocks = static_cast<unsigned>(std::min<long long>((items + 255) / 256, 65535LL * 16));
  dense_delta_kernel<<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(out),
                                             static_cast<const __nv_bfloat16*>(dout), delta, d);
  XP_CHECK_LAUNCH("dense_delta_kernel");
  __nv_bfloat16* dx = static_cast<__nv_bfloat16*>(dqkv);
  dense_bwd_kv_kernel<<<dense_grid(d), DENSE_THREADS, DENSE_BWD_KV_SMEM, st>>>(tm, tdo, lse, delta, dx, d);
  XP_CHECK_LAUNCH("dense_bwd_kv_kernel");
  dense_bwd_q_kernel<<<dense_grid(d), DENSE_THREADS, DENSE_BWD_Q_SMEM, st>>>(tm, tdo, lse, delta, dx, d, q_scale);
  XP_CHECK_LAUNCH("dense_bwd_q_kernel");
  return 0;
}
