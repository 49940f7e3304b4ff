// Fused multi-tensor optimizer step: global-norm gradient clipping + the reference's AdamW ("weight decay fix").
//
// Reference: AdamW.step CLIP-ViP/src/optimization/adamw.py:40-103 and clip_grad_norm_ at pretrain/run_pretrain.py:408-411.
// The reference walks ~300 parameters in Python and launches ~10 elementwise kernels per parameter (mul_, add_, addcmul_,
// sqrt, add_, addcdiv_, add_) plus the norm reductions: ~3000 launches moving each fp32 value many times.  Here the whole
// step is three launches over a device-side tensor table: one read of g for the norm, then one pass that reads
// p, g, m, v and writes p, m, v (28 B/parameter — the HBM roofline of the step: 149.6 M parameters -> 4.2 GB) and can
// also emit the bf16 compute copy the GEMMs consume (saves the separate cast pass).
//
// Arithmetic follows adamw.py's order in fp32: g' = g * coef; m = b1*m + (1-b1)*g'; v = b2*v + (1-b2)*g'*g';
// p -= step_size * m / (sqrt(v) + eps) with eps OUTSIDE the bias correction (step_size = lr*sqrt(1-b2^t)/(1-b1^t) is
// computed by the host per tensor); then the decoupled decay p -= (lr*wd) * p on the updated p.  IEEE sqrt/div
// (the library is built with --use_fast_math, so they are requested explicitly).
#include "../../include/xpretrain_b200.h"
#include "common.h"
#include "ptx.cuh"

namespace xp {

constexpr int OPT_THREADS = 256;
constexpr int OPT_CHUNK = 8192;   // elements per block: 256 threads x 8 x float4

static_assert(sizeof(XpOptTensor) == 64, "XpOptTensor must stay 64 bytes (the host fills it as a packed table)");

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

__global__ void __launch_bounds__(OPT_THREADS)
opt_sumsq_kernel(const XpOptTensor* __restrict__ table, const int2* __restrict__ blocks, float* __restrict__ partial) {
  __shared__ float red[OPT_THREADS / 32];
  const int2 e = blocks[blockIdx.x];
  const XpOptTensor t = table[e.x];
  const long long lo = static_cast<long long>(e.y) * OPT_CHUNK;
  const long long hi = lo + OPT_CHUNK < t.n ? lo + OPT_CHUNK : t.n;
  const float* g = static_cast<const float*>(t.g);
  float acc = 0.f;
  if (aligned16(g)) {
    for (long long i = lo + threadIdx.x * 4; i < hi; i += OPT_THREADS * 4) {
      if (i + 4 <= hi) {
        const float4 v = *reinterpret_cast<const float4*>(g + i);
        acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      } else {
        for (long long j = i; j < hi; ++j) acc += g[j] * g[j];
      }
    }
  } else {
    for (long long i = lo + threadIdx.x; i < hi; i += OPT_THREADS) acc += g[i] * g[i];
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < OPT_THREADS / 32; ++w) s += red[w];
    partial[blockIdx.x] = s;
  }
}

// norm_out[0] = total 2-norm, norm_out[1] = clip coefficient min(1, max_norm / (norm + 1e-6)) (1 when max_norm <= 0).
// One block, fixed summation order in double: deterministic.
__global__ void __launch_bounds__(1024)
opt_norm_finalize_kernel(const float* __restrict__ partial, int n, float max_norm, float* __restrict__ norm_out) {
  __shared__ double red[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 1024) acc += static_cast<double>(partial[i]);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 32; ++w) s += red[w];
    const float total = static_cast<float>(sqrt(s));
    norm_out[0] = total;
    const float coef = max_norm > 0.f ? __fdiv_rn(max_norm, total + 1e-6f) : 1.f;
    // clamp(coef, max=1) as clip_grad_norm_ does it: a NaN norm gives a NaN coefficient, which then reaches every gradient
    norm_out[1] = coef > 1.f ? 1.f : coef;
  }
}

__device__ __forceinline__ void adamw_one(float& p, float g, float& m, float& v, float coef, float b1, float b2, float eps,
                                          float step_size, float decay) {
  const float gs = g * coef;
  m = m * b1 + gs * (1.f - b1);
  v = v * b2 + gs * gs * (1.f - b2);
  const float denom = __fsqrt_rn(v) + eps;
  p = p - step_size * __fdiv_rn(m, denom);
  p = p - decay * p;    // decay == 0 for the no-decay groups
}

template <bool SCALE_ONLY>
__global__ void __launch_bounds__(OPT_THREADS)
opt_adamw_kernel(const XpOptTensor* __restrict__ table, const int2* __restrict__ blocks, const float* __restrict__ coef_ptr,
                 float b1, float b2, float eps) {
  const int2 e = blocks[blockIdx.x];
  const XpOptTensor t = table[e.x];
  const long long lo = static_cast<long long>(e.y) * OPT_CHUNK;
  const long long hi = lo + OPT_CHUNK < t.n ? lo + OPT_CHUNK : t.n;
  const float coef = coef_ptr != nullptr ? coef_ptr[1] : 1.f;
  float* p = static_cast<float*>(t.p);
  float* g = static_cast<float*>(const_cast<void*>(t.g));
  float* m = static_cast<float*>(t.m);
  float* v = static_cast<float*>(t.v);
  __nv_bfloat16* pb = static_cast<__nv_bfloat16*>(t.p_bf16);
  if (SCALE_ONLY) {     // clip_grad_norm_ used on its own: scale the gradients in place
    if (coef >= 1.f) return;
    for (long long i = lo + threadIdx.x; i < hi; i += OPT_THREADS) g[i] *= coef;
    return;
  }
  const bool vec = aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v) && (pb == nullptr || (reinterpret_cast<uintptr_t>(pb) & 7) == 0);
  if (vec) {
    for (long long i = lo + threadIdx.x * 4; i < hi; i += OPT_THREADS * 4) {
      if (i + 4 <= hi) {
        float4 pv = *reinterpret_cast<float4*>(p + i);
        const float4 gv = *reinterpret_cast<const float4*>(g + i);
        float4 mv = *reinterpret_cast<float4*>(m + i);
        float4 vv = *reinterpret_cast<float4*>(v + i);
        adamw_one(pv.x, gv.x, mv.x, vv.x, coef, b1, b2, eps, t.step_size, t.decay);
        adamw_one(pv.y, gv.y, mv.y, vv.y, coef, b1, b2, eps, t.step_size, t.decay);
        adamw_one(pv.z, gv.z, mv.z, vv.z, coef, b1, b2, eps, t.step_size, t.decay);
        adamw_one(pv.w, gv.w, mv.w, vv.w, coef, b1, b2, eps, t.step_size, t.decay);
        *reinterpret_cast<float4*>(p + i) = pv;
        *reinterpret_cast<float4*>(m + i) = mv;
        *reinterpret_cast<float4*>(v + i) = vv;
        if (pb != nullptr)
          *reinterpret_cast<uint2*>(pb + i) = make_uint2(pack_bf16(pv.x, pv.y), pack_bf16(pv.z, pv.w));
      } else {
        for (long long j = i; j < hi; ++j) {
          float pj = p[j], mj = m[j], vj = v[j];
          adamw_one(pj, g[j], mj, vj, coef, b1, b2, eps, t.step_size, t.decay);
          p[j] = pj; m[j] = mj; v[j] = vj;
          if (pb != nullptr) pb[j] = __float2bfloat16(pj);
        }
      }
    }
  } else {
    for (long long j = lo + threadIdx.x; j < hi; j += OPT_THREADS) {
      float pj = p[j], mj = m[j], vj = v[j];
      adamw_one(pj, g[j], mj, vj, coef, b1, b2, eps, t.step_size, t.decay);
      p[j] = pj; m[j] = mj; v[j] = vj;
      if (pb != nullptr) pb[j] = __float2bfloat16(pj);
    }
  }
}

// Multi-tensor fp32 -> bf16 cast / fp32 copy over the same table: row.g = fp32 source, row.p_bf16 = bf16 destination
// (or, when it is null, row.p = fp32 destination).  The models refresh ALL bf16 compute copies of a tower with one launch
// per forward, so weights written behind autograd's back (`p.data.addcdiv_` of the reference AdamW, adamw.py:89,101;
// EMA / checkpoint swaps) can never be stale.  HBM-bound: 6 B per parameter.
__global__ void __launch_bounds__(OPT_THREADS)
opt_cast_kernel(const XpOptTensor* __restrict__ table, const int2* __restrict__ blocks) {
  const int2 e = blocks[blockIdx.x];
  const XpOptTensor t = table[e.x];
  const long long lo = static_cast<long long>(e.y) * OPT_CHUNK;
  const long long hi = lo + OPT_CHUNK < t.n ? lo + OPT_CHUNK : t.n;
  const float* src = static_cast<const float*>(t.g);
  __nv_bfloat16* pb = static_cast<__nv_bfloat16*>(t.p_bf16);
  float* pf = static_cast<float*>(t.p);
  if (pb != nullptr) {
    if (aligned16(src) && (reinterpret_cast<uintptr_t>(pb) & 7) == 0) {
      for (long long i = lo + threadIdx.x * 4; i < hi; i += OPT_THREADS * 4) {
        if (i + 4 <= hi) {
          const float4 v = *reinterpret_cast<const float4*>(src + i);
          *reinterpret_cast<uint2*>(pb + i) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
        } else {
          for (long long j = i; j < hi; ++j) pb[j] = __float2bfloat16(src[j]);
        }
      }
    } else {
      for (long long j = lo + threadIdx.x; j < hi; j += OPT_THREADS) pb[j] = __float2bfloat16(src[j]);
    }
  } else if (pf != nullptr) {
    for (long long j = lo + threadIdx.x; j < hi; j += OPT_THREADS) pf[j] = src[j];
  }
}

}  // namespace xp

using namespace xp;

extern "C" int xp_cast_table(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks, void* stream) {
  XP_ENTER(table_dev);
  if (n_blocks <= 0) return fail("xp_cast_table: empty block map");
  opt_cast_kernel<<<n_blocks, OPT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      table_dev, reinterpret_cast<const int2*>(block_map_dev));
  XP_CHECK_LAUNCH("opt_cast_kernel");
  return 0;
}

extern "C" int32_t xp_opt_chunk_elems(void) { return OPT_CHUNK; }

extern "C" int xp_opt_grad_norm(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks,
                                float* partial_dev, float max_norm, float* norm_out_dev, void* stream) {
  XP_ENTER(table_dev);
  if (n_blocks <= 0) return fail("xp_opt_grad_norm: empty block map");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  opt_sumsq_kernel<<<n_blocks, OPT_THREADS, 0, st>>>(table_dev, reinterpret_cast<const int2*>(block_map_dev), partial_dev);
  XP_CHECK_LAUNCH("opt_sumsq_kernel");
  opt_norm_finalize_kernel<<<1, 1024, 0, st>>>(partial_dev, n_blocks, max_norm, norm_out_dev);
  XP_CHECK_LAUNCH("opt_norm_finalize_kernel");
  return 0;
}

extern "C" int xp_opt_scale_grads(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks,
                                  const float* norm_dev, void* stream) {
  XP_ENTER(table_dev);
  if (n_blocks <= 0) return fail("xp_opt_scale_grads: empty block map");
  if (norm_dev == nullptr) return fail("xp_opt_scale_grads: needs the {norm, coef} pair written by xp_opt_grad_norm");
  opt_adamw_kernel<true><<<n_blocks, OPT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      table_dev, reinterpret_cast<const int2*>(block_map_dev), norm_dev, 0.f, 0.f, 0.f);
  XP_CHECK_LAUNCH("opt_scale_kernel");
  return 0;
}

extern "C" int xp_opt_adamw_step(const XpOptTensor* table_dev, const int32_t* block_map_dev, int32_t n_blocks,
                                 const float* norm_dev, float beta1, float beta2, float eps, void* stream) {
  XP_ENTER(table_dev);
  if (n_blocks <= 0) return fail("xp_opt_adamw_step: empty block map");
  if (!(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f))
    return fail("xp_opt_adamw_step: betas must be in [0, 1) and eps >= 0");   // adamw.py:24-35
  opt_adamw_kernel<false><<<n_blocks, OPT_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      table_dev, reinterpret_cast<const int2*>(block_map_dev), norm_dev, beta1, beta2, eps);
  XP_CHECK_LAUNCH("opt_adamw_kernel");
  return 0;
}
