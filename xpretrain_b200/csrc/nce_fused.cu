// ONE kernel for the contrastive head of a data-parallel step:
//     hvd.allgather(vis), hvd.allgather(txt)            CLIP-ViP/src/pretrain/run_pretrain.py:344-345
//     NCELearnableTempLoss.forward                      CLIP-ViP/src/optimization/loss.py:134-141
// i.e. cross-GPU exchange of the [b, d] embeddings + logit-scale matmul + both softmaxes + loss + dL/dZ, fused:
//
//   1. every rank publishes its fp32 embeddings into its exchange buffer (symmetric memory, mapped by all peers over
//      NVLink / NVSwitch) and raises a per-rank epoch flag on every peer (st.release.sys) — a device-side barrier, no NCCL;
//   2. each CTA owns one 128 x 128 tile of Z = V T^T.  Its producer warps LOAD THE OPERAND ROWS STRAIGHT FROM THE OWNING
//      PEER'S MEMORY (ld.relaxed.sys, 16 B per lane, coalesced per row), split every fp32 value into bf16 hi + lo and
//      stage the four 128B-swizzled operand tiles {A_hi, A_lo, B_hi, B_lo} of a 64-column block in shared memory; each
//      of the two producer warpgroups then issues wgmma for hi*hi + hi*lo + lo*hi on its 64 tile rows into register
//      accumulators (fp32-grade logits on bf16 tensor cores).  A two-stage ring overlaps the NVLink loads of block c+1
//      with the MMAs of block c — the transfer rides under the math tile by tile, there is no gathered copy of the fp32
//      embeddings;
//   3. the epilogue scales by exp(logit_scale), parks the tile in shared memory and emits per-tile row / column
//      (max, sum-exp) partials; after ONE grid barrier every CTA combines the partials it needs into the row / column
//      log-sum-exps and writes its tile of exp(logit_scale) * dL/dZ (bf16) plus its share of the loss and of
//      d logit_scale; the last CTA to finish adds the per-tile shares in a fixed order (deterministic, identical on all ranks).
// Tiles on the first tile column / row also write the bf16 copies of V / T that the (local, collective-free) gradient
// GEMMs dV = s G T, dT = s G^T V consume.  Launched cooperatively: (N/128)^2 co-resident CTAs, one per SM (2-stage ring) or two per SM (compact variant).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

constexpr int NF_THREADS = 256;                    // warpgroup 0: A producers + epilogue, 1: B producers; both issue MMAs
constexpr int NF_TILE = 128;
constexpr int NF_STAGE_BYTES = 4 * NF_TILE * 128;  // A_hi, A_lo, B_hi, B_lo: [128 rows][64 bf16]
constexpr int NF_ZLD = NF_TILE + 1;                // padded row pitch of the parked fp32 tile
// Operand ring (2 stages: NVLink loads of block c+1 overlap the MMAs of block c) or, when (N/128)^2 tiles do not fit one CTA
// per SM, a compact variant with ONE stage, half the loads in flight and <= 128 registers, so that two CTAs share an SM.
// The parked fp32 tile (128 x 129) reuses the ring after the MMAs.
__host__ __device__ constexpr int nf_smem_main(int stages) {
  return stages * NF_STAGE_BYTES > NF_TILE * NF_ZLD * 4 ? stages * NF_STAGE_BYTES : NF_TILE * NF_ZLD * 4;
}
__host__ __device__ constexpr int nf_smem_bytes(int stages) {
  return nf_smem_main(stages) + 2 * NF_TILE * 4 + 8 * 4 + 4 * 8 + 1024;
}
constexpr int NF_FLAG_BYTES = 1024;

struct NfParams {
  const float* vis_local;
  const float* txt_local;
  void* const* peers;
  const float* logit_scale;
  __nv_bfloat16* g;
  __nv_bfloat16* vis_hi;
  __nv_bfloat16* txt_hi;
  float* loss;
  float* dscale;
  float* rowpart;      // [nt][Npad][2]
  float* colpart;      // [nt][Npad][2]
  float* part;         // [nt * nt][2]
  unsigned int* counters;   // [0] published slices, [1] grid barrier, [2] finish ticket
  int rank, world, b, d, N, nt, Npad, mode;
  unsigned int epoch;
  long long ld_g, slot_bytes;
};

__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// peer (NVLink) or local fp32 row segment, never through a stale L1 line
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
// Ranks reach the exchange at different times (a slow rank's forward, the first step's lazy initialisation): the flag wait
// tolerates ~60 s of skew before it traps; the intra-GPU waits keep the library-wide 4 s limit.
constexpr long long NF_PEER_TIMEOUT_CYCLES = 120000000000ll;
__device__ __forceinline__ void spin_guard(long long t0, const char* what, long long limit = XP_WAIT_TIMEOUT_CYCLES) {
  if (clock64() - t0 > limit) {
    printf("xpretrain_b200: nce_gather_fused timeout waiting for %s (block %d thread %d)\n", what, blockIdx.x, threadIdx.x);
    __trap();
  }
}

// source row of global embedding row r: V (which = 0) or T (which = 1)
__device__ __forceinline__ const float* nf_row(const NfParams& p, int which, int r) {
  const int rk = r / p.b, loc = r - rk * p.b;
  if (p.mode == 0) {
    const char* base = static_cast<const char*>(p.peers[rk]) + NF_FLAG_BYTES + (p.epoch & 1u) * p.slot_bytes;
    return reinterpret_cast<const float*>(base) + (static_cast<long long>(which) * p.b + loc) * p.d;
  }
  return static_cast<const float*>(p.peers[which * p.world + rk]) + static_cast<long long>(loc) * p.d;
}

template <int STAGES>
__global__ void __launch_bounds__(NF_THREADS, 3 - STAGES) nce_gather_fused_kernel(const NfParams p) {
  constexpr int NF_SMEM_MAIN = nf_smem_main(STAGES);
  constexpr int LOADS = STAGES == 2 ? 16 : 8;        // 16-byte peer loads in flight per thread
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  float* zs = reinterpret_cast<float*>(gbase);                       // parked tile (after the MMAs retired)
  float* s_lr = reinterpret_cast<float*>(gbase + NF_SMEM_MAIN);      // [128] row LSE
  float* s_lc = s_lr + NF_TILE;                                      // [128] column LSE
  float* s_red = s_lc + NF_TILE;                                     // [8]
  uint64_t* bar = reinterpret_cast<uint64_t*>(s_red + 8);            // full[2], empty[2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tp = blockIdx.x / p.nt, tq = blockIdx.x % p.nt;          // tile row (videos) / tile column (texts)
  const int G = gridDim.x;

  if (tid == 0) {
    mbar_init(&bar[0], 8);
    mbar_init(&bar[1], 8);
    mbar_init(&bar[2], 2);    // one arrival per warpgroup once its MMAs on the stage retired
    mbar_init(&bar[3], 2);
    fence_barrier_init();
  }

  // ---------------------------------------------------------------- 1. publish + device-side flag barrier
  if (p.mode == 0) {
    char* own = static_cast<char*>(p.peers[p.rank]);
    float4* dst = reinterpret_cast<float4*>(own + NF_FLAG_BYTES + (p.epoch & 1u) * p.slot_bytes);
    const int n4 = p.b * p.d / 4;
    for (int i = blockIdx.x * NF_THREADS + tid; i < 2 * n4; i += G * NF_THREADS)
      dst[i] = i < n4 ? reinterpret_cast<const float4*>(p.vis_local)[i] : reinterpret_cast<const float4*>(p.txt_local)[i - n4];
    __threadfence_system();
    __syncthreads();
    if (tid == 0) atomicAdd(&p.counters[0], 1u);
    if (blockIdx.x == 0) {
      if (tid == 0) {
        const long long t0 = clock64();
        while (ld_acquire_gpu(&p.counters[0]) < static_cast<unsigned int>(G)) spin_guard(t0, "local publish");
        __threadfence_system();
      }
      __syncthreads();
      if (tid < p.world)      // raise this rank's flag on every peer (and on itself)
        st_release_sys(reinterpret_cast<unsigned int*>(p.peers[tid]) + p.rank, p.epoch);
    }
    if (tid < p.world) {
      const unsigned int* flag = reinterpret_cast<const unsigned int*>(own) + tid;
      const long long t0 = clock64();
      while (static_cast<int>(ld_acquire_sys(flag) - p.epoch) < 0) spin_guard(t0, "a peer's epoch flag", NF_PEER_TIMEOUT_CYCLES);
    }
  }
  __syncthreads();

  // ---------------------------------------------------------------- 2. logits tile on wgmma, operands from peer memory
  const int nblk = p.d / 64;
  float acc[64];                                     // rows [64 which, 64 which + 64) x 128 columns of the tile
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  {
    const int which = warp >> 2;                     // 0: A = V rows of tile row tp, 1: B = T rows of tile column tq
    const int pw = warp & 3;
    const int tile0 = (which == 0 ? tp : tq) * NF_TILE;
    const bool write_hi = which == 0 ? (tq == 0) : (tp == 0);
    __nv_bfloat16* hi_out = which == 0 ? p.vis_hi : p.txt_hi;
    const int sub = lane >> 4, t16 = lane & 15;      // 2 rows per warp instruction, 16 lanes x 16 B per 256-B row segment
    for (int c = 0; c < nblk; ++c) {
      const int s = c % STAGES;
      const uint32_t ph = (c / STAGES) & 1;
      mbar_wait_nocall(&bar[2 + s], ph ^ 1);
      const uint32_t st_hi = base + s * NF_STAGE_BYTES + which * 2 * NF_TILE * 128, st_lo = st_hi + NF_TILE * 128;
#pragma unroll
      for (int it0 = 0; it0 < 16; it0 += LOADS) {
      float4 x[LOADS];
#pragma unroll
      for (int it = 0; it < LOADS; ++it) {           // LOADS NVLink loads in flight before the first use
        const int r = tile0 + (it0 + it) * 8 + pw * 2 + sub;
        x[it] = r < p.N ? ld_peer_f4(nf_row(p, which, r) + c * 64 + t16 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int it = 0; it < LOADS; ++it) {
        const int row = (it0 + it) * 8 + pw * 2 + sub;
        const float v[4] = {x[it].x, x[it].y, x[it].z, x[it].w};
        float h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          h[e] = __bfloat162float(__float2bfloat16(v[e]));
          l[e] = v[e] - h[e];
        }
        const uint32_t h0 = pack_bf16(h[0], h[1]), h1 = pack_bf16(h[2], h[3]);
        const uint32_t l0 = pack_bf16(l[0], l[1]), l1 = pack_bf16(l[2], l[3]);
        const uint32_t off = row * 128 + (((t16 >> 1) ^ (row & 7)) << 4) + (t16 & 1) * 8;
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(st_hi + off), "r"(h0), "r"(h1) : "memory");
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(st_lo + off), "r"(l0), "r"(l1) : "memory");
        const int r = tile0 + row;
        if (write_hi && r < p.N)
          *reinterpret_cast<uint2*>(hi_out + static_cast<long long>(r) * p.d + c * 64 + t16 * 4) = make_uint2(h0, h1);
      }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&bar[s]);
      // both operand tiles of block c staged (8 warps): this warpgroup's 64 rows of A against all 128 rows of B
      mbar_wait_nocall(&bar[s], ph);
      const uint32_t a_hi = base + s * NF_STAGE_BYTES + which * 64 * 128, a_lo = a_hi + NF_TILE * 128,
                     b_hi = base + s * NF_STAGE_BYTES + 2 * NF_TILE * 128, b_lo = b_hi + NF_TILE * 128;
      const uint32_t aa[3] = {a_hi, a_hi, a_lo}, bb[3] = {b_hi, b_lo, b_hi};
      wgmma_fence_regs(acc);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_m64n128k16_bf16<0, 0>(acc, make_smem_desc_sw128(aa[g] + ks * 32, 16, 1024),
                                      make_smem_desc_sw128(bb[g] + ks * 32, 16, 1024));
      wgmma_commit();
      wgmma_fence_regs(acc);
      if (STAGES == 2) {
        wgmma_wait<1>();                             // block c-1's MMAs retired: its stage may be refilled
        if (c > 0 && (tid & 127) == 0) mbar_arrive(&bar[2 + (s ^ 1)]);
      } else {
        wgmma_wait<0>();                             // the single stage is free once this block's MMAs retired
        if ((tid & 127) == 0) mbar_arrive(&bar[2]);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
  }

  // ---------------------------------------------------------------- 3a. epilogue: scaled tile -> smem, per-tile partials
  const float s_exp = expf(*p.logit_scale);
  const int rows_valid = min(NF_TILE, p.N - tp * NF_TILE), cols_valid = min(NF_TILE, p.N - tq * NF_TILE);
  __syncthreads();                                   // every MMA has read the ring: the parked tile may overwrite it
  {
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int col = i * 8 + (lane & 3) * 2;
      zs[r0 * NF_ZLD + col] = s_exp * acc[4 * i];
      zs[r0 * NF_ZLD + col + 1] = s_exp * acc[4 * i + 1];
      zs[(r0 + 8) * NF_ZLD + col] = s_exp * acc[4 * i + 2];
      zs[(r0 + 8) * NF_ZLD + col + 1] = s_exp * acc[4 * i + 3];
    }
  }
  __syncthreads();
  if (warp < 4) {
    float m = -INFINITY, sum = 0.f;
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      const float* o = zs + tid * NF_ZLD + ch * 32;
      float cm = -INFINITY;
#pragma unroll
      for (int e = 0; e < 32; ++e)
        if (ch * 32 + e < cols_valid) cm = fmaxf(cm, o[e]);
      if (cm > m) {
        sum *= expf(m - cm);
        m = cm;
      }
#pragma unroll
      for (int e = 0; e < 32; ++e)
        if (ch * 32 + e < cols_valid) sum += expf(o[e] - m);
    }
    if (tid < rows_valid) {
      float* rp = p.rowpart + (static_cast<long long>(tq) * p.Npad + tp * NF_TILE + tid) * 2;
      rp[0] = m;
      rp[1] = sum;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (tid < cols_valid) {                           // thread = column: partial over this tile's rows
      float cm = -INFINITY;
      for (int i = 0; i < rows_valid; ++i) cm = fmaxf(cm, zs[i * NF_ZLD + tid]);
      float cs = 0.f;
      for (int i = 0; i < rows_valid; ++i) cs += expf(zs[i * NF_ZLD + tid] - cm);
      float* cp = p.colpart + (static_cast<long long>(tp) * p.Npad + tq * NF_TILE + tid) * 2;
      cp[0] = cm;
      cp[1] = cs;
    }
    __threadfence();
  }
  // ---------------------------------------------------------------- grid barrier: every tile's partials are visible
  __syncthreads();
  if (tid == 0) {
    atomicAdd(&p.counters[1], 1u);
    const long long t0 = clock64();
    while (ld_acquire_gpu(&p.counters[1]) < static_cast<unsigned int>(G)) spin_guard(t0, "the grid barrier");
  }
  __syncthreads();

  // ---------------------------------------------------------------- 3b. LSEs, gradient tile, loss / d logit_scale shares
  if (warp < 4) {
    {
      float m = -INFINITY;
      const int gi = tp * NF_TILE + tid, gj = tq * NF_TILE + tid;
      float lr = 0.f, lc = 0.f;
      if (tid < rows_valid) {
        for (int k = 0; k < p.nt; ++k) m = fmaxf(m, __ldcg(p.rowpart + (static_cast<long long>(k) * p.Npad + gi) * 2));
        float sacc = 0.f;
        for (int k = 0; k < p.nt; ++k) {
          const float* rp = p.rowpart + (static_cast<long long>(k) * p.Npad + gi) * 2;
          sacc += __ldcg(rp + 1) * expf(__ldcg(rp) - m);
        }
        lr = m + logf(sacc);
      }
      if (tid < cols_valid) {
        m = -INFINITY;
        for (int k = 0; k < p.nt; ++k) m = fmaxf(m, __ldcg(p.colpart + (static_cast<long long>(k) * p.Npad + gj) * 2));
        float sacc = 0.f;
        for (int k = 0; k < p.nt; ++k) {
          const float* cp = p.colpart + (static_cast<long long>(k) * p.Npad + gj) * 2;
          sacc += __ldcg(cp + 1) * expf(__ldcg(cp) - m);
        }
        lc = m + logf(sacc);
      }
      s_lr[tid] = lr;
      s_lc[tid] = lc;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const float inv_n = 1.f / static_cast<float>(p.N);
    float dsc = 0.f, lterm = 0.f;
    if (tid < cols_valid) {                           // thread = column: coalesced bf16 stores along each row of G
      const int gj = tq * NF_TILE + tid;
      const float lc = s_lc[tid];
      for (int i = 0; i < rows_valid; ++i) {
        const int gi = tp * NF_TILE + i;
        const float z = zs[i * NF_ZLD + tid];
        const float g = (expf(z - s_lr[i]) + expf(z - lc) - (gi == gj ? 2.f : 0.f)) * inv_n;
        dsc += g * z;
        p.g[static_cast<long long>(gi) * p.ld_g + gj] = __float2bfloat16(g * s_exp);
      }
      if (tp == tq) lterm = (s_lr[tid] + lc - 2.f * zs[tid * NF_ZLD + tid]) * inv_n;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dsc += __shfl_xor_sync(0xffffffffu, dsc, o);
      lterm += __shfl_xor_sync(0xffffffffu, lterm, o);
    }
    if (lane == 0) {
      s_red[warp] = dsc;
      s_red[4 + warp] = lterm;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if (tid == 0) {
      p.part[blockIdx.x * 2] = (s_red[4] + s_red[5]) + (s_red[6] + s_red[7]);
      p.part[blockIdx.x * 2 + 1] = (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]);
      __threadfence();
      const unsigned int ticket = atomicAdd(&p.counters[2], 1u);
      if (ticket == static_cast<unsigned int>(G) - 1u) {     // last tile: fixed-order sum -> the same bits on every rank
        __threadfence();
        float l = 0.f, ds = 0.f;
        for (int k = 0; k < G; ++k) {
          l += __ldcg(p.part + 2 * k);
          ds += __ldcg(p.part + 2 * k + 1);
        }
        *p.loss = l;
        *p.dscale = ds;
        p.counters[0] = 0u;
        p.counters[1] = 0u;
        p.counters[2] = 0u;
      }
    }
  }
}

}  // namespace xp

using namespace xp;

extern "C" int64_t xp_nce_gather_exchange_bytes(int32_t b, int32_t d, int32_t world) {
  (void)world;
  return NF_FLAG_BYTES + 2LL * 2 * b * d * static_cast<int64_t>(sizeof(float));
}

extern "C" int64_t xp_nce_gather_workspace_bytes(int32_t N) {
  const int64_t nt = (N + NF_TILE - 1) / NF_TILE, npad = nt * NF_TILE;
  return (2 * nt * npad * 2 + nt * nt * 2) * static_cast<int64_t>(sizeof(float)) + 64;
}

extern "C" int xp_nce_gather_fused(const XpNceGather* a, void* stream) {
  XP_ENTER(a->g_scaled);
  if (a->world < 1 || a->rank < 0 || a->rank >= a->world) return fail("xp_nce_gather_fused: bad rank / world");
  if (a->world > 256) return fail("xp_nce_gather_fused: at most 256 ranks (one flag word per rank in the 1 KiB flag block)");
  if (a->d % 64 != 0 || a->d < 64) return fail("xp_nce_gather_fused: embedding width must be a multiple of 64");
  if (a->b < 1) return fail("xp_nce_gather_fused: empty batch");
  const long long N = static_cast<long long>(a->world) * a->b;
  const int nt = static_cast<int>((N + NF_TILE - 1) / NF_TILE);
  // every tile's CTA must be co-resident (one grid barrier): one CTA per SM with the 2-stage ring, else two per SM with the
  // compact variant (N <= 1408 / 2048 on the 132 SMs of an H100)
  static int blocks_per_sm[2] = {0, 0};   // [0]: compact (1 stage), [1]: 2 stages
  if (blocks_per_sm[1] == 0) {
    const void* k1 = reinterpret_cast<const void*>(nce_gather_fused_kernel<1>);
    const void* k2 = reinterpret_cast<const void*>(nce_gather_fused_kernel<2>);
    XP_CHECK_CUDA(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, nf_smem_bytes(1)));
    XP_CHECK_CUDA(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, nf_smem_bytes(2)));
    XP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm[0], k1, NF_THREADS, nf_smem_bytes(1)));
    XP_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm[1], k2, NF_THREADS, nf_smem_bytes(2)));
  }
  const bool two_stage = nt * nt <= blocks_per_sm[1] * sm_count();
  if (!two_stage && nt * nt > blocks_per_sm[0] * sm_count())
    return fail("xp_nce_gather_fused: global batch too large for one co-resident wave of 128x128 tiles");
  if (a->ld_g < N) return fail("xp_nce_gather_fused: ld_g < N");
  if (a->mode == 0 && (a->b * a->d) % 4 != 0) return fail("xp_nce_gather_fused: b*d must be a multiple of 4");
  NfParams p;
  p.vis_local = a->vis_local; p.txt_local = a->txt_local;
  p.peers = a->peer_bufs; p.logit_scale = a->logit_scale;
  p.g = static_cast<__nv_bfloat16*>(a->g_scaled);
  p.vis_hi = static_cast<__nv_bfloat16*>(a->vis_hi); p.txt_hi = static_cast<__nv_bfloat16*>(a->txt_hi);
  p.loss = a->loss; p.dscale = a->d_logit_scale;
  p.rank = a->rank; p.world = a->world; p.b = a->b; p.d = a->d; p.N = static_cast<int>(N); p.nt = nt; p.Npad = nt * NF_TILE;
  p.mode = a->mode; p.epoch = a->epoch; p.ld_g = a->ld_g;
  p.slot_bytes = 2LL * a->b * a->d * static_cast<long long>(sizeof(float));
  float* ws = a->workspace;
  p.rowpart = ws;
  p.colpart = ws + 2LL * nt * p.Npad;
  p.part = ws + 4LL * nt * p.Npad;
  p.counters = reinterpret_cast<unsigned int*>(ws + 4LL * nt * p.Npad + 2LL * nt * nt);
  void* args[] = {&p};
  const void* kern = two_stage ? reinterpret_cast<const void*>(nce_gather_fused_kernel<2>)
                               : reinterpret_cast<const void*>(nce_gather_fused_kernel<1>);
  XP_CHECK_CUDA(cudaLaunchCooperativeKernel(kern, dim3(nt * nt), dim3(NF_THREADS), args, nf_smem_bytes(two_stage ? 2 : 1),
                                            static_cast<cudaStream_t>(stream)));
  XP_CHECK_LAUNCH("nce_gather_fused_kernel");
  return 0;
}
