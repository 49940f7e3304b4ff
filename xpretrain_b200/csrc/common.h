// Host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <string>
#include <type_traits>

#include "../../include/xpretrain_b200.h"

namespace xp {

void set_error(const std::string& msg);
int fail(const std::string& msg);  // records msg, returns -1
extern std::atomic<int64_t> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count();  // SMs of the current device (cached per device)

// 2-D bf16 tensor map with 128-byte swizzle.  inner/outer are extents in
// elements, row_stride in elements, box = {box_inner, box_outer}.
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride,
                      uint32_t box_inner, uint32_t box_outer);
// 3-D bf16 tensor map with 128-byte swizzle: extents {inner, mid, outer} in elements, strides of the mid and outer
// dimensions in elements, box = {box_inner, box_mid, 1}.  Box rows past `mid` read as zero (TMA out-of-bounds fill).
int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t mid, uint64_t outer,
                      uint64_t row_stride, uint64_t mid_stride, uint32_t box_inner, uint32_t box_mid);

// Bind the CUDA context that owns `device_ptr` to the calling thread if the thread has none.  PyTorch runs
// autograd backward on worker threads that may not have touched CUDA yet; this library links its own
// (static) runtime, so without this a first call from such a thread would see "no current context" (or
// silently use device 0 on a multi-GPU rank).
int ensure_context(const void* device_ptr);
#define XP_ENTER(ptr)                                   \
  do {                                                  \
    if (::xp::ensure_context(ptr) != 0) return -1;      \
  } while (0)

#define XP_CHECK_CUDA(expr)                                                                         \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) return ::xp::fail(std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

#define XP_CHECK_LAUNCH(name)                                                                             \
  do {                                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                                  \
    if (_e != cudaSuccess) return ::xp::fail(std::string(name) + " launch: " + cudaGetErrorString(_e)); \
    ::xp::count_launch();                                                                                 \
  } while (0)

inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Raises kernel K's dynamic shared-memory limit to `bytes` on the first call (once per process); 0 or -1 as fail().
template <auto K>
int smem_limit(int bytes) {
  static bool done = false;
  if (!done) {
    XP_CHECK_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done = true;
  }
  return 0;
}

// Runtime value -> template argument: f(std::integral_constant<int, V>{}) for the V in Vs equal to v, else fail(what).
template <int... Vs, class F>
int dispatch(int v, const char* what, F&& f) {
  int rc = 0;
  const bool found = ((v == Vs && (rc = f(std::integral_constant<int, Vs>{}), true)) || ...);
  return found ? rc : fail(what);
}

// Element type of an XP_DTYPE_* code, and f(T{}) for the element type T of `dtype` (fail(what) for another code).
template <int D>
using dtype_t = std::conditional_t<D == XP_DTYPE_F32, float, std::conditional_t<D == XP_DTYPE_BF16, __nv_bfloat16, __half>>;
template <class F>
int dispatch_dtype(int dtype, const char* what, F&& f) {
  return dispatch<XP_DTYPE_F32, XP_DTYPE_BF16, XP_DTYPE_F16>(dtype, what, [&](auto d) { return f(dtype_t<d.value>{}); });
}

}  // namespace xp
