// Dense (non-causal, unmasked) multi-head attention, head_dim 64, over sequences of consecutive rows of the fused
// token-major qkv buffer: the joint space-time and space-only attentions of HD-VILA's TimeSformer (Attention.forward,
// timesformer.py:156-173, on x of shape [B, H*W*T, C] or [B*T, H*W, C], :202-205).  See xp_dense_attention_* in
// include/xpretrain_b200.h for the ABI.
//
// Runs the streamed pipeline of attn_wgmma.cuh with a three-stage ring, one CTA per two 64-row tiles of one (sequence,
// head).  delta = rowsum(dO * O) is computed by a small kernel ahead of the two backward kernels, whose producer warpgroup
// loads it with the LSE.
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
#include "attn_wgmma.cuh"

namespace xp {

namespace {

struct DenseDims {
  long long n_rows, ld_qkv, ld_o;
  int H, n_seq, L, C;
};

// Layout of a CTA of grid (ceil(ntiles / 2), H, n_seq): the 64-row tiles of sequence blockIdx.z.
struct Dense {
  static constexpr int STAGES = 3;
  static constexpr bool ZERO_FILL = true;   // 3-D tensor map: box rows past the sequence end read as zero
  DenseDims d;

  __device__ void bind() {}
  __device__ int h() const { return blockIdx.y; }
  __device__ long long row0() const { return static_cast<long long>(blockIdx.z) * d.L; }   // first row of the sequence
  __device__ int ntiles() const { return (d.L + ATILE - 1) / ATILE; }
  __device__ int rows(int j) const { return min(ATILE, d.L - j * ATILE); }
  __device__ bool skip(int, int) const { return false; }
  __device__ void load(void* dst, const CUtensorMap* tm, uint64_t* bar, int m, int j) const {
    tma_load_3d(dst, tm, bar, m * d.C + h() * HD, j * ATILE, blockIdx.z);
  }
  __device__ __nv_bfloat16* row(__nv_bfloat16* base, long long ld, int j, int i) const {
    return base + (row0() + j * ATILE + i) * ld + h() * HD + (threadIdx.x & 3) * 2;
  }
};

struct DenseFwd : Dense {
  __nv_bfloat16* out;
  float* lse;

  __device__ void store_fwd(int qt, int i, int r, const float (&o)[32], float m, float l) const {
    const float inv = 1.f / l;   // > 0: every query sees at least one key
    __nv_bfloat16* dst = row(out, d.ld_o, qt, i);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      *reinterpret_cast<uint32_t*>(dst + k * 8) = pack_bf16(o[4 * k + 2 * r] * inv, o[4 * k + 2 * r + 1] * inv);
    if ((threadIdx.x & 3) == 0) lse[static_cast<long long>(h()) * d.n_rows + row0() + qt * ATILE + i] = m + logf(l);
  }
};

struct DenseBwd : Dense {
  const float* lse;
  const float* delta;
  __nv_bfloat16* dqkv;
  float q_scale;

  // threads 0-63: lse, 64-127: delta.  Rows past the end: lse = +inf gives P = 0 exactly (their Q and dO are
  // zero-filled, so every product is finite)
  __device__ void fill_stats(float* s, int qb) const {
    const int i = threadIdx.x & 63, which = threadIdx.x >> 6;
    const float* src = (which == 0 ? lse : delta) + static_cast<long long>(h()) * d.n_rows + row0();
    const bool valid = i < rows(qb);
    const float v = valid ? __ldg(src + qb * ATILE + i) : 0.f;
    s[which * ATILE + i] = which == 0 ? (valid ? v * LOG2E : INFINITY) : v;
  }
  // +inf / 0 past the end: P = 0
  __device__ void row_stats(int qt, int q_lo, float (&lse_r)[2], float (&del_r)[2]) const {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int i = q_lo + r * 8;
      const long long at = static_cast<long long>(h()) * d.n_rows + row0() + qt * ATILE + i;
      lse_r[r] = i < rows(qt) ? __ldg(lse + at) * LOG2E : INFINITY;
      del_r[r] = i < rows(qt) ? __ldg(delta + at) : 0.f;
    }
  }
  __device__ void store_kv(int kt, int key, int r, const float (&dk)[32], const float (&dv)[32]) const {
    __nv_bfloat16* dst = row(dqkv, d.ld_qkv, kt, key);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      *reinterpret_cast<uint32_t*>(dst + d.C + k * 8) = pack_bf16(dk[4 * k + 2 * r], dk[4 * k + 2 * r + 1]);
      *reinterpret_cast<uint32_t*>(dst + 2 * d.C + k * 8) = pack_bf16(dv[4 * k + 2 * r], dv[4 * k + 2 * r + 1]);
    }
  }
  __device__ void store_q(int qt, int q, int r, const float (&dq)[32]) const {
    __nv_bfloat16* dst = row(dqkv, d.ld_qkv, qt, q);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      *reinterpret_cast<uint32_t*>(dst + k * 8) = pack_bf16(dq[4 * k + 2 * r] * q_scale, dq[4 * k + 2 * r + 1] * q_scale);
  }
};

}  // namespace

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

namespace {
constexpr int DENSE_FWD_SMEM = stream_fwd_smem(Dense::STAGES);
constexpr int DENSE_BWD_KV_SMEM = stream_kv_smem(Dense::STAGES);
constexpr int DENSE_BWD_Q_SMEM = stream_q_smem(Dense::STAGES);

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
  const int ntiles = (d.L + ATILE - 1) / ATILE;
  return dim3((ntiles + 1) / 2, d.H, d.n_seq);
}

// {columns, seq_len, n_seq} view of a token-major [rows, ld] buffer: box rows past a sequence's end read as zero
int seq_tmap(CUtensorMap* tm, const void* base, long long ld, const DenseDims& d) {
  return make_tmap_bf16_3d(tm, base, ld, d.L, d.n_seq, ld, ld * d.L, HD, ATILE);
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
  if (smem_limit<stream_fwd_kernel<DenseFwd>>(DENSE_FWD_SMEM)) return -1;
  const DenseFwd p{{d}, static_cast<__nv_bfloat16*>(out), lse};
  stream_fwd_kernel<<<dense_grid(d), STREAM_THREADS, DENSE_FWD_SMEM, static_cast<cudaStream_t>(stream)>>>(tm, p);
  XP_CHECK_LAUNCH("dense_fwd_kernel");
  return 0;
}

extern "C" int xp_dense_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                                      void* dqkv, const XpDenseAttn* desc, float q_scale, void* stream) {
  XP_ENTER(qkv);
  DenseDims d;
  if (int rc = to_dims(desc, d, "xp_dense_attention_bwd")) return rc;
  if (!aligned(out, 16)) return fail("xp_dense_attention_bwd: out must be 16-byte aligned");
  CUtensorMap tm, tdo;
  if (seq_tmap(&tm, qkv, d.ld_qkv, d) || seq_tmap(&tdo, dout, d.ld_o, d)) return -1;
  if (smem_limit<stream_bwd_kv_kernel<DenseBwd>>(DENSE_BWD_KV_SMEM) ||
      smem_limit<stream_bwd_q_kernel<DenseBwd>>(DENSE_BWD_Q_SMEM))
    return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long items = static_cast<long long>(d.n_seq) * d.L * d.H * 8;
  const unsigned blocks = static_cast<unsigned>(std::min<long long>((items + 255) / 256, 65535LL * 16));
  dense_delta_kernel<<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(out),
                                             static_cast<const __nv_bfloat16*>(dout), delta, d);
  XP_CHECK_LAUNCH("dense_delta_kernel");
  const DenseBwd p{{d}, lse, delta, static_cast<__nv_bfloat16*>(dqkv), q_scale};
  stream_bwd_kv_kernel<<<dense_grid(d), STREAM_THREADS, DENSE_BWD_KV_SMEM, st>>>(tm, tdo, p);
  XP_CHECK_LAUNCH("dense_bwd_kv_kernel");
  stream_bwd_q_kernel<<<dense_grid(d), STREAM_THREADS, DENSE_BWD_Q_SMEM, st>>>(tm, tdo, p);
  XP_CHECK_LAUNCH("dense_bwd_q_kernel");
  return 0;
}
