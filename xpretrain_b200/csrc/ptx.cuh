// sm_90a PTX wrappers used by the kernels of this library: mbarrier, TMA
// (cp.async.bulk.tensor), warpgroup MMA (wgmma) and its shared-memory
// descriptors.  Hand-written for H100; nothing here is portable to other
// architectures and nothing here is meant to be.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace xp {

#ifndef XP_WAIT_TIMEOUT_CYCLES
// A stuck mbarrier wait traps instead of hanging the GPU (≈4 s at 2 GHz).
#define XP_WAIT_TIMEOUT_CYCLES (8000000000ll)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// ----------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > XP_WAIT_TIMEOUT_CYCLES) {
      printf("xpretrain_b200: mbarrier wait timeout (block %d thread %d parity %u)\n", blockIdx.x, threadIdx.x,
             parity);
      __trap();
    }
  }
}
// The same wait without the printf: for waits between asynchronous wgmma groups, where a function call would make
// ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > XP_WAIT_TIMEOUT_CYCLES) __trap();
  }
}

// ---------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// TMA store: a 128B-swizzled shared-memory box -> global memory (bulk async group of the issuing thread).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups are still READING their shared-memory source
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// -------------------------------------------------------------------- wgmma
// Warpgroup MMA (sm_90a): the four warps of a warpgroup issue together; accumulators live in registers.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] += A[64 x 16] * B[16 x 128]^T, bf16 operands from shared-memory descriptors, fp32 accumulators.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.  Accumulator layout (per warp w of the
// warpgroup, lane l): d[4i + {0,1}] = row 16w + l/4, columns 8i + 2(l%4) + {0,1}; d[4i + {2,3}] = the same, row + 8.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, 1, 1, 1, %66, %67;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB));
}

// D[64 x 64] += A[64 x 16] * B[16 x 64]^T with both operands from shared-memory descriptors (TA / TB = 1: MN-major).
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, 1, 1, 1, %34, %35;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB));
}
// Same with A from registers: a[4] is the m16k16 bf16 fragment of this warp's 16 rows (the layout of an accumulator's
// column pair packed per 16 columns: {row, k 0-7}, {row + 8, k 0-7}, {row, k 8-15}, {row + 8, k 8-15}).
template <int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, {%32, %33, %34, %35}, %36, 1, 1, 1, %37;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "n"(TB));
}

// ------------------------------------------------------- warpgroup registers / named barriers
// Move per-thread registers between the warpgroups of a CTA (sm_90a).  Every warp of the warpgroup executes it; the
// count is a multiple of 8 in [24, 256].
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// Named barrier `id` (1-15; 0 is __syncthreads) over `threads` threads: bar.sync waits, bar.arrive only counts.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor, sm_90 wgmma format (cute/arch/mma_sm90_desc.hpp documents the bit layout):
// start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | layout [62,64) with SWIZZLE_128B = 1.
// K-major 128B-swizzled tiles: SBO = 1024 (8-row groups), LBO unused.  MN-major: LBO = stride of the 64-element
// MN atoms, SBO = stride of the 8-k-row groups.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ------------------------------------------------------------------- misc
// Transpose a 4 x 4 matrix of 32-bit words held by the four lanes of each quad (lanes 4m .. 4m + 3): afterwards lane q
// holds in v[j] what lane j held in v[q].  Every lane of the warp must call it.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4]) {
  const int q = threadIdx.x & 3;
  uint32_t out[4];
  out[0] = out[1] = out[2] = out[3] = 0u;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int j = q ^ t;   // the partner lane: it wants my v[j], I want its v[q]
    const uint32_t send = j == 0 ? v[0] : j == 1 ? v[1] : j == 2 ? v[2] : v[3];
    const uint32_t got = t == 0 ? send : __shfl_xor_sync(0xffffffffu, send, t);
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c == j) out[c] = got;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) v[c] = out[c];
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

// ------------------------------------------------------- 8-wide conversions
// Eight consecutive elements <-> float[8]: one 16-byte access for bf16 / fp16, two for fp32.
__device__ __forceinline__ void unpack8_bf16(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8_bf16(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16(f[0], f[1]); u.y = pack_bf16(f[2], f[3]); u.z = pack_bf16(f[4], f[5]); u.w = pack_bf16(f[6], f[7]);
  return u;
}
__device__ __forceinline__ void unpack8_f16(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 v = __half22float2(h[i]);
    f[2 * i] = v.x;
    f[2 * i + 1] = v.y;
  }
}
// Saturating: a value beyond fp16's range becomes +-65504, not inf (the row kernels' fp16 residual stream, DESIGN §3).
__device__ __forceinline__ uint4 pack8_f16_satfinite(const float (&f)[8]) {
  uint4 u;
  uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(w[i]) : "f"(f[2 * i + 1]), "f"(f[2 * i]));
  return u;
}
__device__ __forceinline__ void load8(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  unpack8_bf16(*reinterpret_cast<const uint4*>(p), f);
}
__device__ __forceinline__ void load8(const __half* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  unpack8_f16(u, f);
}
__device__ __forceinline__ void store8(float* p, const float (&f)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = pack8_bf16(f);
}
__device__ __forceinline__ void store8_satfinite(__half* p, const float (&f)[8]) {
  *reinterpret_cast<uint4*>(p) = pack8_f16_satfinite(f);
}

// Scalar conversions (round to nearest; fp16 overflows to inf).
template <typename T>
__device__ __forceinline__ float to_f32(T v) { return static_cast<float>(v); }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16(v); }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half(v); }

// ------------------------------------------------------- warp reductions
// Over all 32 lanes, xor butterfly: every lane gets the result.
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// sigmoid(y) = 0.5 + 0.5 * tanh(y / 2): ONE MUFU op (tanh.approx) instead of ex2 + rcp — the GELU epilogues of
// the fc1 GEMMs issue many MUFU ops per output element.  tanh.approx is good to ~2^-11, below bf16's 2^-9.
__device__ __forceinline__ float fast_sigmoid(float y) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * y));
  return fmaf(0.5f, t, 0.5f);
}
// QuickGELU = x * sigmoid(1.702 x) (transformers QuickGELUActivation, selected at CLIP_ViP.py:389)
__device__ __forceinline__ float quick_gelu(float x) { return x * fast_sigmoid(1.702f * x); }
// y is clamped to [-64, 64]: beyond |y| ~ 17 the fp32 sigmoid is already exactly 0 or 1, so no finite result changes,
// but for |x| >~ 2e38 (within bf16 range) the unclamped 1.702 x overflows and y * (1 - s) becomes inf * 0 = NaN.
// Comparisons rather than fminf / fmaxf, so that a NaN x still gives NaN.
__device__ __forceinline__ float quick_gelu_grad(float x) {
  float y = 1.702f * x;
  y = y > 64.f ? 64.f : (y < -64.f ? -64.f : y);
  const float s = fast_sigmoid(y);
  return s * fmaf(y, 1.f - s, 1.f);
}

}  // namespace xp
