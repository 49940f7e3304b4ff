#include "common.h"

#include <mutex>

#include "../../include/xpretrain_b200.h"

namespace xp {

static thread_local std::string t_error;
std::atomic<int64_t> g_launches{0};

void set_error(const std::string& msg) { t_error = msg; }
int fail(const std::string& msg) {
  t_error = msg;
  return -1;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    // The driver symbol is resolved through the runtime so the library does not link libcuda.
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

typedef CUresult (*CtxGetCurrentFn)(CUcontext*);
typedef CUresult (*CtxSetCurrentFn)(CUcontext);
typedef CUresult (*PointerGetAttributeFn)(void*, CUpointer_attribute, CUdeviceptr);

static void* driver_symbol(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
    return nullptr;
  return p;
}

int ensure_context(const void* device_ptr) {
  static thread_local bool bound = false;
  if (bound) return 0;
  static CtxGetCurrentFn get_cur = reinterpret_cast<CtxGetCurrentFn>(driver_symbol("cuCtxGetCurrent"));
  static CtxSetCurrentFn set_cur = reinterpret_cast<CtxSetCurrentFn>(driver_symbol("cuCtxSetCurrent"));
  static PointerGetAttributeFn ptr_attr =
      reinterpret_cast<PointerGetAttributeFn>(driver_symbol("cuPointerGetAttribute"));
  if (!get_cur || !set_cur || !ptr_attr)
    return fail("CUDA driver unavailable (no GPU): this library has no CPU path");
  CUcontext cur = nullptr;
  if (get_cur(&cur) == CUDA_SUCCESS && cur != nullptr) {
    bound = true;
    return 0;
  }
  if (device_ptr == nullptr) return fail("null device pointer");
  CUcontext owner = nullptr;
  if (ptr_attr(&owner, CU_POINTER_ATTRIBUTE_CONTEXT, reinterpret_cast<CUdeviceptr>(device_ptr)) == CUDA_SUCCESS &&
      owner != nullptr) {
    if (set_cur(owner) != CUDA_SUCCESS) return fail("cuCtxSetCurrent failed");
  } else {
    // pool / stream-ordered allocations report no owning context: fall back to the device ordinal
    int ordinal = -1;
    if (ptr_attr(&ordinal, CU_POINTER_ATTRIBUTE_DEVICE_ORDINAL, reinterpret_cast<CUdeviceptr>(device_ptr)) !=
            CUDA_SUCCESS ||
        ordinal < 0)
      return fail("cannot find the CUDA device of the first pointer argument (is it a device pointer?)");
    if (cudaSetDevice(ordinal) != cudaSuccess) return fail("cudaSetDevice failed");
  }
  bound = true;
  return 0;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride,
                      uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail("cuTensorMapEncodeTiled unavailable (no CUDA driver / no GPU): this library has no CPU path");
  if (!aligned(base, 16)) return fail("tensor map: base pointer must be 16-byte aligned");
  if ((row_stride * 2) % 16 != 0) return fail("tensor map: row stride must be a multiple of 8 bf16 elements");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {row_stride * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(int(r)));
  return 0;
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t mid, uint64_t outer,
                      uint64_t row_stride, uint64_t mid_stride, uint32_t box_inner, uint32_t box_mid) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail("cuTensorMapEncodeTiled unavailable (no CUDA driver / no GPU): this library has no CPU path");
  if (!aligned(base, 16)) return fail("tensor map: base pointer must be 16-byte aligned");
  if ((row_stride * 2) % 16 != 0 || (mid_stride * 2) % 16 != 0)
    return fail("tensor map: strides must be multiples of 8 bf16 elements");
  cuuint64_t dims[3] = {inner, mid, outer};
  cuuint64_t strides[2] = {row_stride * 2, mid_stride * 2};
  cuuint32_t box[3] = {box_inner, box_mid, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(int(r)));
  return 0;
}

}  // namespace xp

extern "C" {
int xp_version(void) { return XP_ABI_VERSION; }
const char* xp_last_error(void) { return xp::t_error.c_str(); }
int64_t xp_launch_count(void) { return xp::g_launches.load(); }
void xp_launch_count_reset(void) { xp::g_launches.store(0); }
}
