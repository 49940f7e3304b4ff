// Video-proxy (ViP) attention for frames longer than the staged kernel of vip_attention.cu takes (M + L > 208): ViT-L/14
// has L = 256 patches per frame at 224 px, 576 at 336 px and 1024 at 448 px.  Same maths (CLIPAttention.forward2,
// CLIP_ViP.py:332-381), same outputs and the same per-frame partials of the global rows as vip_attention.cu, whose combine
// kernels finish both paths.
//
// A frame is too long to stage whole (a TMA box holds at most 256 rows), so it runs the streamed pipeline of
// attn_wgmma.cuh with a two-stage ring, one CTA per two 64-row tiles of one (b, h, t).  The rows of one (b, h, t) are cut
// into tiles of 64: tiles j < nft = ceil(L / 64) hold frame rows [64 j, 64 j + 64) (rows past L are masked; TMA reads
// whatever follows, or zero fill at the end of the tensor), and tile nft holds the M global rows (rows past M masked).
// Patch queries of frame t see every key tile of frame t plus the global tile; global queries see the same keys, except
// that the global keys count only in frame 0, so that global x global pairs enter once.  delta = rowsum(dO * O) is
// computed inside the backward kernels: by the producer warpgroup for the key-stationary kernel, by each consumer quad
// for the query-stationary kernel.
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "attn_wgmma.cuh"
#include "vip_attention.h"

namespace xp {

namespace {

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

// Layout of a CTA of grid (ceil((nft + 1) / 2), T, B*H): the nft frame tiles of (b, t), then the global tile.
struct VipLong {
  static constexpr int STAGES = 2;
  static constexpr bool ZERO_FILL = false;   // a frame tile's dead rows are the next frame's rows
  AttnDims d;
  int b_;   // blockIdx.z / H, resolved once by bind(): not re-derived after every barrier wait

  __device__ void bind() { b_ = blockIdx.z / d.H; }
  __device__ int t() const { return blockIdx.y; }
  __device__ int h() const { return blockIdx.z - b_ * d.H; }
  __device__ int b() const { return b_; }
  __device__ long long bh() const { return blockIdx.z; }   // b * H + h
  __device__ int nft() const { return (d.L + ATILE - 1) / ATILE; }
  __device__ int ntiles() const { return nft() + 1; }
  __device__ int rows(int j) const { return j < nft() ? min(ATILE, d.L - j * ATILE) : d.M; }
  __device__ bool skip(int qt, int kt) const { return qt == nft() && kt == nft() && t() != 0; }
  // sequence index (within the sample) of row i of tile j
  __device__ long long seq(int j, int i) const {
    return j < nft() ? d.M + static_cast<long long>(t()) * d.L + static_cast<long long>(j) * ATILE + i : i;
  }
  __device__ void load(void* dst, const CUtensorMap* tm, uint64_t* bar, int m, int j) const {
    tma_load_2d(dst, tm, bar, m * d.C + h() * HD, static_cast<int>(static_cast<long long>(b()) * d.S + seq(j, 0)));
  }
  // global-row partials of this frame: part [.., M, 66] (forward), gpart [.., M, 3, 64] (backward)
  __device__ float* frame_part(float* base, int width) const { return base + (bh() * d.T + t()) * d.M * width; }
};

struct VipLongFwd : VipLong {
  __nv_bfloat16* out;
  float* lse;
  float* part;

  __device__ void store_fwd(int qt, int row, int r, const float (&o)[32], float m, float l) const {
    const int lane = threadIdx.x & 31;
    if (qt == nft()) {   // global-query row: this frame's partial (fp32, unnormalised)
      float* p = frame_part(part, 66) + row * 66;
      if ((lane & 3) == 0) {
        p[0] = m;
        p[1] = l;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        p[2 + i * 8 + (lane & 3) * 2] = o[4 * i + 2 * r];
        p[2 + i * 8 + (lane & 3) * 2 + 1] = o[4 * i + 2 * r + 1];
      }
    } else {             // frame row: normalised output + LSE
      const float inv = l > 0.f ? 1.f / l : 0.f;
      const long long sq = seq(qt, row);
      __nv_bfloat16* dst = out + (static_cast<long long>(b()) * d.S + sq) * d.ld_o + h() * HD + (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + i * 8) = pack_bf16(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
      if ((lane & 3) == 0) lse[bh() * d.S + sq] = m + logf(l);
    }
  }
};

struct VipLongBwd : VipLong {
  const __nv_bfloat16* out;
  const __nv_bfloat16* dout;
  const float* lse;
  __nv_bfloat16* dqkv;
  float* gpart;
  float q_scale;

  __device__ long long o_off(long long sq) const { return (static_cast<long long>(b()) * d.S + sq) * d.ld_o + h() * HD; }

  // two threads per query row, 32 columns each
  __device__ void fill_stats(float* s, int qb) const {
    const int row = threadIdx.x >> 1, half = threadIdx.x & 1;
    const bool valid = row < rows(qb);
    float dot = 0.f;
    long long sq = 0;
    if (valid) {
      sq = seq(qb, row);
      const long long off = o_off(sq) + half * 32;
      dot = dot16(dout + off, out + off) + dot16(dout + off + 16, out + off + 16);
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    if (half == 0) {
      s[row] = valid ? lse[bh() * d.S + sq] * LOG2E : INFINITY;
      s[ATILE + row] = dot;
    }
  }
  // the four lanes of a quad each sum 16 columns of delta
  __device__ void row_stats(int qt, int q_lo, float (&lse_r)[2], float (&del_r)[2]) const {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = q_lo + r * 8;
      float dot = 0.f;
      lse_r[r] = INFINITY;
      if (row < rows(qt)) {
        const long long sq = seq(qt, row);
        const long long off = o_off(sq) + (lane & 3) * 16;
        dot = dot16(dout + off, out + off);
        lse_r[r] = lse[bh() * d.S + sq] * LOG2E;
      }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      del_r[r] = dot;
    }
  }
  __device__ __nv_bfloat16* dqkv_row(int j, int i) const {
    return dqkv + (static_cast<long long>(b()) * d.S + seq(j, i)) * d.ld_qkv + h() * HD + (threadIdx.x & 3) * 2;
  }
  __device__ float* gpart_row(int i) const {
    return frame_part(gpart, 3 * HD) + static_cast<long long>(i) * 3 * HD + (threadIdx.x & 3) * 2;
  }

  __device__ void store_kv(int kt, int key, int r, const float (&dk)[32], const float (&dv)[32]) const {
    if (kt != nft()) {
      __nv_bfloat16* row = dqkv_row(kt, key);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        *reinterpret_cast<uint32_t*>(row + d.C + i * 8) = pack_bf16(dk[4 * i + 2 * r], dk[4 * i + 2 * r + 1]);
        *reinterpret_cast<uint32_t*>(row + 2 * d.C + i * 8) = pack_bf16(dv[4 * i + 2 * r], dv[4 * i + 2 * r + 1]);
      }
    } else {
      float* g = gpart_row(key);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        g[HD + i * 8] = dk[4 * i + 2 * r]; g[HD + i * 8 + 1] = dk[4 * i + 2 * r + 1];
        g[2 * HD + i * 8] = dv[4 * i + 2 * r]; g[2 * HD + i * 8 + 1] = dv[4 * i + 2 * r + 1];
      }
    }
  }
  __device__ void store_q(int qt, int q, int r, const float (&dq)[32]) const {
    if (qt != nft()) {
      __nv_bfloat16* row = dqkv_row(qt, q);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(row + i * 8) = pack_bf16(dq[4 * i + 2 * r] * q_scale, dq[4 * i + 2 * r + 1] * q_scale);
    } else {
      float* g = gpart_row(q);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        g[i * 8] = dq[4 * i + 2 * r];
        g[i * 8 + 1] = dq[4 * i + 2 * r + 1];
      }
    }
  }
};

int long_grid(const AttnDims& d, dim3& grid) {
  const long long bh = static_cast<long long>(d.B) * d.H;
  if (d.T > 65535 || bh > 65535) return fail("vip_attention: T and B*H must be <= 65535");
  if (static_cast<long long>(d.B) * d.S > 0x7fffffffLL) return fail("vip_attention: B*S must fit in int32");
  const int ntiles = (d.L + ATILE - 1) / ATILE + 1;
  grid = dim3((ntiles + 1) / 2, d.T, static_cast<unsigned>(bh));
  return 0;
}

constexpr int LONG_FWD_SMEM = stream_fwd_smem(VipLong::STAGES);
constexpr int LONG_BWD_KV_SMEM = stream_kv_smem(VipLong::STAGES);
constexpr int LONG_BWD_Q_SMEM = stream_q_smem(VipLong::STAGES);

}  // namespace

int vip_long_attn_fwd(const AttnDims& d, const void* qkv, void* out, float* lse, float* part, cudaStream_t st) {
  dim3 grid;
  if (long_grid(d, grid)) return -1;
  CUtensorMap tm;
  if (make_tmap_bf16_2d(&tm, qkv, d.ld_qkv, static_cast<uint64_t>(d.B) * d.S, d.ld_qkv, HD, ATILE)) return -1;
  if (smem_limit<stream_fwd_kernel<VipLongFwd>>(LONG_FWD_SMEM)) return -1;
  const VipLongFwd p{{d, 0}, static_cast<__nv_bfloat16*>(out), lse, part};
  stream_fwd_kernel<<<grid, STREAM_THREADS, LONG_FWD_SMEM, st>>>(tm, p);
  XP_CHECK_LAUNCH("vip_long_fwd_kernel");
  return 0;
}

int vip_long_attn_bwd(const AttnDims& d, const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                      float* gpart, float q_scale, cudaStream_t st) {
  dim3 grid;
  if (long_grid(d, grid)) return -1;
  CUtensorMap tm, tdo;
  const uint64_t rows = static_cast<uint64_t>(d.B) * d.S;
  if (make_tmap_bf16_2d(&tm, qkv, d.ld_qkv, rows, d.ld_qkv, HD, ATILE) ||
      make_tmap_bf16_2d(&tdo, dout, d.ld_o, rows, d.ld_o, HD, ATILE))
    return -1;
  if (smem_limit<stream_bwd_kv_kernel<VipLongBwd>>(LONG_BWD_KV_SMEM) ||
      smem_limit<stream_bwd_q_kernel<VipLongBwd>>(LONG_BWD_Q_SMEM))
    return -1;
  const VipLongBwd p{{d, 0}, static_cast<const __nv_bfloat16*>(out), static_cast<const __nv_bfloat16*>(dout), lse,
                     static_cast<__nv_bfloat16*>(dqkv), gpart, q_scale};
  stream_bwd_kv_kernel<<<grid, STREAM_THREADS, LONG_BWD_KV_SMEM, st>>>(tm, tdo, p);
  XP_CHECK_LAUNCH("vip_long_bwd_kv_kernel");
  stream_bwd_q_kernel<<<grid, STREAM_THREADS, LONG_BWD_Q_SMEM, st>>>(tm, tdo, p);
  XP_CHECK_LAUNCH("vip_long_bwd_q_kernel");
  return 0;
}

}  // namespace xp
