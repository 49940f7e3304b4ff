// Persistent warp-specialised bf16 GEMM for sm_90a:
//   TMA (cp.async.bulk.tensor, 128B swizzle) -> shared-memory ring (full / empty mbarriers)
//   -> wgmma (two consumer warpgroups, fp32 accumulators in registers)
//   -> register epilogue (bias / q-scale / QuickGELU / dQuickGELU / GELU / residual) -> global.
// One CTA per SM, 3 warpgroups: warpgroup 0 = TMA producer (one thread, 40 registers), warpgroups 1-2 = MMA + epilogue
// (232 registers).  Two schedules, chosen per launch in xp_gemm:
//   BN = 128, ping-pong: each consumer owns whole 128 x 128 tiles, alternately; one consumer's epilogue runs while the
//     other's k-loop keeps the tensor cores busy.
//   BN = 256, cooperative: both consumers split each 128 x 256 tile by rows ([0, 64) and [64, 128)); while they run
//     its epilogue the producer is already filling the ring with the next tile's k-blocks.
//
// Replaces (see include/xpretrain_b200.h) every nn.Linear forward/backward on
// the CLIP-ViP hot path: CLIP_ViP.py:341-343,379,393-395,1141-1145 and the
// patch-embedding conv :178 (as an im2col GEMM).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"
#include <cstdlib>

namespace xp {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = one 128-byte swizzle row
constexpr int MMA_K = 16;
constexpr int GEMM_THREADS = 384;  // producer warpgroup + 2 consumer warpgroups

struct GemmDev {
  void* c;
  const float* bias;
  const __nv_bfloat16* residual;
  __nv_bfloat16* aux;
  int M, N, K;
  long long ldc, ldr, ld_aux;
  long long c_group, c_group_stride, r_group, r_group_stride;
  int act;
  int splits;
  int scale_cols;
  float alpha, col_scale;
  uint32_t mn_lbo, mn_sbo;  // MN-major descriptor strides (bytes): 64-element atom stride, 8-k-row group stride
};

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  // ring + 1 KiB alignment slack + barriers
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
};

__device__ __forceinline__ float act_gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float act_gelu_erf_grad(float x) {
  float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
  float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

template <int BN, int A_MN, int B_MN, int OUT, int ACT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  // BN = 128, ping-pong: a consumer owns whole 128 x 128 tiles, accumulator block mh = rows [64 mh, 64 mh + 64).
  // BN = 256, cooperative: the consumers split each 128 x 256 tile by rows, accumulator block h = columns
  // [128 h, 128 h + 128) of the consumer's 64 rows.
  constexpr bool PINGPONG = BN == 128;
  constexpr int MH = PINGPONG ? 2 : 1;  // 64-row accumulator blocks per consumer thread
  constexpr int NH = BN / 128;          // n128 accumulator blocks per consumer thread
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_mn = num_m * num_n;
  const int total = num_mn * p.splits;
  const int kb_total = (p.K + BK - 1) / BK;
  const int kb_per = (kb_total + p.splits - 1) / p.splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PINGPONG ? 1 : 2);  // one arrival per consumer warpgroup reading the stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int split = tile / num_mn;
        const int mn = tile - split * num_mn;
        const int m_blk = mn / num_n;
        const int n_blk = mn - m_blk * num_n;
        const int k0 = split * kb_per;
        const int k1 = min(kb_total, k0 + kb_per);
        for (int kb = k0; kb < k1; ++kb) {
          mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
          uint8_t* sA = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sB = sA + Cfg::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
          if (A_MN) {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)
              tma_load_2d(sA + i * (BK * 128), &tmA, &full_bar[stage], m_blk * BM + i * 64, kb * BK);
          } else {
            tma_load_2d(sA, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
          }
          if (B_MN) {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_2d(sB + i * (BK * 128), &tmB, &full_bar[stage], n_blk * BN + i * 64, kb * BK);
          } else {
            tma_load_2d(sB, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ---------------------------------------------- MMA + epilogue
    setmaxnreg_inc<232>();
    const int cw = wg - 1;                    // consumer warpgroup 0 / 1
    const int wq = (threadIdx.x >> 5) & 3;    // warp within the warpgroup: 16 rows of each 64-row block
    // kernel parameters used per element live in registers
    constexpr int act = ACT;
    const int N = p.N, scale_cols = p.scale_cols;
    const float alpha = p.alpha, col_scale = p.col_scale;
    __nv_bfloat16* const aux_p = p.aux;
    constexpr bool need_aux_in = (ACT == XP_ACT_DQUICK_GELU || ACT == XP_ACT_DGELU_ERF);
    // the one extra bf16 INPUT the epilogue reads: the saved pre-activation (dGELU) or the residual
    const __nv_bfloat16* const xin_p = need_aux_in ? p.aux : p.residual;
    // one 64-row A slab = one 64-element MN atom (MN-major) or 64 swizzled 128-byte rows (K-major)
    constexpr uint32_t A_OFF = 64 * 128;
    // ping-pong turn: the consumers' k-loops alternate in tile order, so that one consumer's epilogue runs while the
    // other's wgmmas keep the tensor cores busy.  Consumer c waits on named barrier 1 + c; the other consumer arrives
    // on it once it has issued its tile's last wgmmas.  The turn also orders the ring: a consumer reaches a stage's
    // fill only after every earlier fill of that stage has been waited for, so its parity wait cannot alias.
    const int cta_tiles = (total - blockIdx.x + gridDim.x - 1) / gridDim.x;
    int stage = 0;
    uint32_t phase = 0;
    int local = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++local) {
      const int split = tile / num_mn;
      const int mn = tile - split * num_mn;
      const int m_blk = mn / num_n;
      const int n_blk = mn - m_blk * num_n;
      const int k0 = split * kb_per;
      const int k1 = min(kb_total, k0 + kb_per);
      if (PINGPONG && (local & 1) != cw) {  // the other consumer's tile: step over its k-blocks in the ring
        const int next = stage + max(0, k1 - k0);
        phase ^= (next / STAGES) & 1;
        stage = next % STAGES;
        continue;
      }
      if (PINGPONG && local > 0) named_bar_sync(1 + cw, 256);
      const bool pass_turn = PINGPONG && local + 1 < cta_tiles;
      if (k0 >= k1) {  // an empty trailing split: nothing to add
        if (pass_turn) named_bar_arrive(2 - cw, 256);
        continue;
      }
      float acc[MH * NH][64];
#pragma unroll
      for (int q = 0; q < MH * NH; ++q)
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[q][i] = 0.f;
      int prev_stage = -1;
      for (int kb = k0; kb < k1; ++kb) {
        mbar_wait_nocall(&full_bar[stage], phase);
        const uint32_t sA = smem_u32(smem + stage * Cfg::STAGE_BYTES) + (PINGPONG ? 0 : cw * A_OFF);
        const uint32_t sB = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
#pragma unroll
        for (int q = 0; q < MH * NH; ++q) wgmma_fence_regs(acc[q]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < BK / MMA_K; ++j) {
#pragma unroll
          for (int mh = 0; mh < MH; ++mh) {
            // K-major: 16 elements = 32 B further along the swizzled row; 8-row groups 1024 B apart.
            // MN-major: 16 k-rows = 2048 B further; 64-element MN atoms BK*128 B apart.
            const uint32_t am = sA + mh * A_OFF;
            const uint64_t adesc = A_MN ? make_smem_desc_sw128(am + j * (MMA_K * 128), p.mn_lbo, p.mn_sbo)
                                        : make_smem_desc_sw128(am + j * (MMA_K * 2), 16, 1024);
#pragma unroll
            for (int h = 0; h < NH; ++h) {
              // columns [128 h, 128 h + 128) of B: two MN atoms (MN-major) or 128 rows (K-major) further, 16 KiB either way
              const uint32_t bh = sB + h * (128 * 128);
              const uint64_t bdesc = B_MN ? make_smem_desc_sw128(bh + j * (MMA_K * 128), p.mn_lbo, p.mn_sbo)
                                          : make_smem_desc_sw128(bh + j * (MMA_K * 2), 16, 1024);
              wgmma_m64n128k16_bf16<A_MN, B_MN>(acc[mh * NH + h], adesc, bdesc);
            }
          }
        }
        wgmma_commit();
#pragma unroll
        for (int q = 0; q < MH * NH; ++q) wgmma_fence_regs(acc[q]);
        // the previous k-block's MMAs have retired once at most this block's group is in flight: free its slot
        wgmma_wait<1>();
        if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      // every wgmma of this tile is issued: the other consumer's k-loop may start while these drain
      if (pass_turn) named_bar_arrive(2 - cw, 256);
      const auto load_bias = [&](float2(&b)[16], int h) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int n = n_blk * BN + h * 128 + i * 8 + (lane & 3) * 2;
          b[i] = make_float2(0.f, 0.f);
          if (p.bias != nullptr && split == 0 && n < N) b[i] = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        }
      };
      // A ping-pong tile is one n128 block wide: its bias is loaded once, while the MMAs drain.  The cooperative tile's
      // two blocks, and the dGELU epilogues' extra registers, do not fit next to the accumulators: those load the bias
      // per row batch below.
      constexpr bool bias_once = PINGPONG && !need_aux_in;
      float2 bias_tile[16];
      if (bias_once) load_bias(bias_tile, 0);
      wgmma_wait<0>();
#pragma unroll
      for (int q = 0; q < MH * NH; ++q) wgmma_fence_regs(acc[q]);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);

      // ---- epilogue straight from the accumulator registers: per 64-row block this thread holds rows r and r + 8,
      // column pairs.  What it reads is loaded in batches ahead of the math and the stores: a load cannot be moved above
      // a store that may alias it, so one load per element would wait out a full memory latency each time.
      // bias, q-scale and the activation of one column pair; returns the bf16 pre-activation the forward GELUs save
      const auto apply = [&](float& v0, float& v1, int n, uint32_t xg) -> uint32_t {
        if (n < scale_cols) {
          v0 *= col_scale;
          v1 *= col_scale;
        }
        uint32_t pre = 0;
        if (act == XP_ACT_QUICK_GELU) {
          pre = pack_bf16(v0, v1);
          v0 = quick_gelu(v0);
          v1 = quick_gelu(v1);
        } else if (act == XP_ACT_DQUICK_GELU) {
          v0 *= quick_gelu_grad(bf16_lo(xg));
          v1 *= quick_gelu_grad(bf16_hi(xg));
        } else if (act == XP_ACT_GELU_ERF) {
          pre = pack_bf16(v0, v1);
          v0 = act_gelu_erf(v0);
          v1 = act_gelu_erf(v1);
        } else if (act == XP_ACT_DGELU_ERF) {
          v0 *= act_gelu_erf_grad(bf16_lo(xg));
          v1 *= act_gelu_erf_grad(bf16_hi(xg));
        } else if (xin_p != nullptr) {   // residual add (never combined with a dGELU epilogue)
          v0 += bf16_lo(xg);
          v1 += bf16_hi(xg);
        }
        return pre;
      };
      constexpr bool save_pre = (ACT == XP_ACT_QUICK_GELU || ACT == XP_ACT_GELU_ERF);
      const int quad = lane & 3;
#pragma unroll
      for (int mh = 0; mh < MH; ++mh) {
        const int row_base = m_blk * BM + (PINGPONG ? mh : cw) * 64 + wq * 16 + (lane >> 2);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int row = row_base + rr * 8;
          // no early exit for rows past M: the bf16 path below shuffles across the warp, so only memory is predicated
          const bool row_ok = row < p.M;
          const long long c_off = p.c_group > 0 ? (row / p.c_group) * p.c_group_stride + (row % p.c_group) * p.ldc
                                                : static_cast<long long>(row) * p.ldc;
          const long long x_off = need_aux_in ? static_cast<long long>(row) * p.ld_aux
                                              : (p.r_group > 0 ? (row / p.r_group) * p.r_group_stride + (row % p.r_group) * p.ldr
                                                               : static_cast<long long>(row) * p.ldr);
          const long long a_off = static_cast<long long>(row) * p.ld_aux;
#pragma unroll
          for (int h = 0; h < NH; ++h) {
            const float* const a = acc[mh * NH + h];
            const int n_h = n_blk * BN + h * 128;
            float2 bias2[16];
            if (bias_once) {
#pragma unroll
              for (int i = 0; i < 16; ++i) bias2[i] = bias_tile[i];
            } else {
              load_bias(bias2, h);
            }
            if (OUT == XP_OUT_BF16) {
              // The four lanes of a quad hold one row's 8-column blocks i as column pairs.  Transposed across the quad,
              // lane q moves all of block 4k + q, so every load and store is 16 bytes and a warp covers whole sectors.
              uint32_t xin[4][4];
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int n8 = n_h + (4 * k + quad) * 8;
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if (xin_p != nullptr && row_ok && n8 < N) v = *reinterpret_cast<const uint4*>(xin_p + x_off + n8);
                xin[k][0] = v.x;
                xin[k][1] = v.y;
                xin[k][2] = v.z;
                xin[k][3] = v.w;
                if (xin_p != nullptr) quad_transpose(xin[k]);
              }
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                uint32_t out[4], pre[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const int i = 4 * k + j;
                  float v0 = fmaf(a[4 * i + 2 * rr], alpha, bias2[i].x);
                  float v1 = fmaf(a[4 * i + 2 * rr + 1], alpha, bias2[i].y);
                  pre[j] = apply(v0, v1, n_h + i * 8 + quad * 2, xin[k][j]);
                  out[j] = pack_bf16(v0, v1);
                }
                const int n8 = n_h + (4 * k + quad) * 8;   // N % 8 == 0: an 8-column block is wholly inside or outside
                quad_transpose(out);
                if (row_ok && n8 < N)
                  *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(p.c) + c_off + n8) =
                      make_uint4(out[0], out[1], out[2], out[3]);
                if (save_pre && aux_p != nullptr) {
                  quad_transpose(pre);
                  if (row_ok && n8 < N)
                    *reinterpret_cast<uint4*>(aux_p + a_off + n8) = make_uint4(pre[0], pre[1], pre[2], pre[3]);
                }
              }
            } else if (row_ok) {   // fp32 outputs (no activation): column pairs
              uint32_t xin[16];
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const int n = n_h + i * 8 + quad * 2;
                xin[i] = 0;
                if (xin_p != nullptr && n < N) xin[i] = *reinterpret_cast<const uint32_t*>(xin_p + x_off + n);
              }
#pragma unroll
              for (int i = 0; i < 16; ++i) {
                const int n = n_h + i * 8 + quad * 2;
                if (n >= N) continue;   // N % 8 == 0: a column pair is either wholly inside or wholly outside
                float v0 = fmaf(a[4 * i + 2 * rr], alpha, bias2[i].x);
                float v1 = fmaf(a[4 * i + 2 * rr + 1], alpha, bias2[i].y);
                apply(v0, v1, n, xin[i]);
                if (OUT == XP_OUT_F32) {
                  *reinterpret_cast<float2*>(static_cast<float*>(p.c) + c_off + n) = make_float2(v0, v1);
                } else {
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(static_cast<float*>(p.c) + c_off + n),
                               "f"(v0), "f"(v1)
                               : "memory");
                }
              }
            }
          }
        }
      }
    }
  }
}

static int g_dbg_mn_lbo = 0, g_dbg_mn_sbo = 0;
}  // namespace xp

// Debug hook for tools/gemm_selftest (not part of the public ABI).
extern "C" void xp_debug_gemm_mn_desc(int lbo, int sbo) {
  xp::g_dbg_mn_lbo = lbo;
  xp::g_dbg_mn_sbo = sbo;
}

extern "C" int xp_gemm(const XpGemm* g, void* stream_v) {
  using namespace xp;
  if (!g) return fail("xp_gemm: null args");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (g->M <= 0 || g->N <= 0 || g->K <= 0) return fail("xp_gemm: M, N, K must be positive");
  if (g->N % 8 != 0) return fail("xp_gemm: N must be a multiple of 8");
  if (!g->a || !g->b || !g->c) return fail("xp_gemm: null operand");
  XP_ENTER(g->a);
  const int splits = g->splits <= 0 ? 1 : g->splits;
  if (splits > 1 && g->out != XP_OUT_F32_ATOMIC) return fail("xp_gemm: split-K requires XP_OUT_F32_ATOMIC");
  if ((g->act == XP_ACT_DQUICK_GELU || g->act == XP_ACT_DGELU_ERF) && !g->aux)
    return fail("xp_gemm: dGELU epilogue needs aux (the forward pre-activation)");
  if (g->act != XP_ACT_NONE && g->out != XP_OUT_BF16) return fail("xp_gemm: activation epilogues need a bf16 output");
  // The epilogue adds a residual only after no activation, addresses aux as plain rows, and tests `n < scale_cols` once
  // per column pair: the combinations below would silently compute something else, so they are refused.
  if (g->act != XP_ACT_NONE && g->residual)
    return fail("xp_gemm: a residual add cannot be combined with an activation epilogue");
  if (g->aux && g->c_group > 0) return fail("xp_gemm: aux cannot be combined with grouped rows (c_group > 0)");
  if (g->scale_cols < 0 || g->scale_cols % 2) return fail("xp_gemm: scale_cols must be even and non-negative");
  const int elem_c = g->out == XP_OUT_BF16 ? 2 : 4;
  if (!aligned(g->c, 16) || (g->ldc * elem_c) % 16)
    return fail("xp_gemm: C must be 16-byte aligned with a 16-byte multiple row pitch");
  if (g->bias && !aligned(g->bias, 16)) return fail("xp_gemm: bias must be 16-byte aligned");
  if (g->residual && (!aligned(g->residual, 16) || (g->ldr % 8)))
    return fail("xp_gemm: residual must be 16-byte aligned, ldr % 8 == 0");
  if (g->aux && (!aligned(g->aux, 16) || (g->ld_aux % 8)))
    return fail("xp_gemm: aux must be 16-byte aligned, ld_aux % 8 == 0");
  if ((g->c_group > 0 && g->c_group_stride % 8) || (g->r_group > 0 && g->r_group_stride % 8))
    return fail("xp_gemm: c_group_stride / r_group_stride must be multiples of 8 elements");

  const int nsm = sm_count();
  const int num_m = static_cast<int>((g->M + BM - 1) / BM);
  int bn = g->block_n;
  if (bn == 0) {
    // Ping-pong 128 x 128 tiles overlap one tile's epilogue with the next tile's k-loop.  That wins where the k-loop is
    // short next to the epilogue: the K-major-B (forward) launches with at most 16 k-blocks per tile.  Everywhere else
    // the cooperative 128 x 256 tiles are faster (measured on H100 SXM, tools/gemm_bench.py): they load a third fewer
    // operand bytes per MMA, which the long k-loops (fc2, dgrad, the split-K wgrad) are bound by.
    const long long tiles256 = static_cast<long long>(num_m) * ((g->N + 255) / 256) * splits;
    const long long kb_split = ((g->K + BK - 1) / BK + splits - 1) / splits;
    const bool short_k_fwd = g->b_layout == 0 && kb_split <= 16;
    bn = (g->N >= 256 && tiles256 >= nsm && !short_k_fwd) ? 256 : 128;
  }
  const char* bad_bn = "xp_gemm: block_n must be 0, 128 or 256";
  if (bn != 128 && bn != 256) return fail(bad_bn);
  // sm_90 has no CTA pairs: cta_pair 0 (auto) and 1 (never) both run the single-CTA kernel
  if (g->cta_pair < 0 || g->cta_pair > 1) return fail("xp_gemm: cta_pair must be 0 or 1 (no CTA pairs on sm_90)");
  const long long total = static_cast<long long>(num_m) * ((g->N + bn - 1) / bn) * splits;
  int grid = g->max_ctas > 0 ? g->max_ctas : nsm;
  if (grid < 1) grid = 1;
  if (grid > total) grid = static_cast<int>(total);

  CUtensorMap tmA, tmB;
  int rc;
  if (g->a_layout == 0)
    rc = make_tmap_bf16_2d(&tmA, g->a, g->K, g->M, g->lda, BK, BM);
  else
    rc = make_tmap_bf16_2d(&tmA, g->a, g->M, g->K, g->lda, 64, BK);
  if (rc) return rc;
  if (g->b_layout == 0)
    rc = make_tmap_bf16_2d(&tmB, g->b, g->K, g->N, g->ldb, BK, bn);
  else
    rc = make_tmap_bf16_2d(&tmB, g->b, g->N, g->K, g->ldb, 64, BK);
  if (rc) return rc;

  GemmDev dev;
  dev.c = g->c;
  dev.bias = g->bias;
  dev.residual = static_cast<const __nv_bfloat16*>(g->residual);
  dev.aux = static_cast<__nv_bfloat16*>(g->aux);
  dev.M = static_cast<int>(g->M);
  dev.N = static_cast<int>(g->N);
  dev.K = static_cast<int>(g->K);
  dev.ldc = g->ldc;
  dev.ldr = g->ldr;
  dev.ld_aux = g->ld_aux;
  dev.c_group = g->c_group;
  dev.c_group_stride = g->c_group_stride;
  dev.r_group = g->r_group;
  dev.r_group_stride = g->r_group_stride;
  dev.act = g->act;
  dev.splits = splits;
  dev.scale_cols = g->scale_cols;
  dev.alpha = g->alpha;
  dev.col_scale = g->col_scale;
  dev.mn_lbo = g_dbg_mn_lbo ? g_dbg_mn_lbo : BK * 128;
  dev.mn_sbo = g_dbg_mn_sbo ? g_dbg_mn_sbo : 1024;

  const char* bad_layout = "xp_gemm: a_layout/b_layout must be 0 or 1";
  auto launch = [&](auto tile_n, auto out, auto act) {
    return dispatch<0, 1>(g->a_layout, bad_layout, [&](auto a_mn) {
      return dispatch<0, 1>(g->b_layout, bad_layout, [&](auto b_mn) {
        constexpr auto kern = gemm_kernel<tile_n.value, a_mn.value, b_mn.value, out.value, act.value>;
        constexpr int smem = GemmCfg<tile_n.value>::SMEM_BYTES;
        if (smem_limit<kern>(smem)) return -1;
        kern<<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, dev);
        XP_CHECK_LAUNCH("gemm_kernel");
        return 0;
      });
    });
  };
  // The activation epilogues exist for bf16 outputs only (forward activations / their gradients).
  using no_act = std::integral_constant<int, XP_ACT_NONE>;
  return dispatch<256, 128>(bn, bad_bn, [&](auto tile_n) {
    return dispatch<XP_OUT_BF16, XP_OUT_F32, XP_OUT_F32_ATOMIC>(g->out, "xp_gemm: bad out mode", [&](auto out) {
      if constexpr (out.value != XP_OUT_BF16)
        return launch(tile_n, out, no_act{});
      else
        return dispatch<XP_ACT_NONE, XP_ACT_QUICK_GELU, XP_ACT_DQUICK_GELU, XP_ACT_GELU_ERF, XP_ACT_DGELU_ERF>(
            g->act, "xp_gemm: bad act", [&](auto act) { return launch(tile_n, out, act); });
    });
  });
}
