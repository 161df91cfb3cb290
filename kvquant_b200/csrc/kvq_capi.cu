// kvquant_b200 -- C-ABI bookkeeping entry points (version, error strings, launch counter) and the host helpers every
// launcher shares (TMA descriptor of a packed cache, SM count).
#include "kvq_common.cuh"
#include <dlfcn.h>

namespace kvq {
unsigned long long g_launch_count = 0;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_cache_tensor_map(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_cols,
                          uint32_t box_rows, int swizzle_bytes) {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    // resolve the driver entry point directly (no link-time dependency on libcuda; the library must load on
    // GPU-less build hosts so that its exports can be checked there)
    void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return (int)cudaErrorInsufficientDriver;
    void* sym = dlsym(h, "cuTensorMapEncodeTiled");
    if (!sym) return (int)cudaErrorNotSupported;
    fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {cols * 4};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE),
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

int num_sms_cached() {
  static int g_sms[64];   // per device (one process may drive several GPUs, see PerDeviceOnce)
  int dev = 0;
  cudaGetDevice(&dev);
  int& n = g_sms[dev & 63];
  if (!n) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace kvq

extern "C" {

int kvq_abi_version(void) { return KVQ_ABI_VERSION; }

uint64_t kvq_launch_count(void) { return kvq::g_launch_count; }

const char* kvq_error_string(int code) {
  switch (code) {
    case 0: return "ok";
    case KVQ_E_BITS: return "kvquant_b200: bits must be 2, 3 or 4";
    case KVQ_E_SHAPE: return "kvquant_b200: inconsistent sizes";
    case KVQ_E_NULL: return "kvquant_b200: required pointer is NULL";
    case KVQ_E_ALIGN: return "kvquant_b200: alignment requirement violated (cache 16 B, Lmax % 4 == 0, LUT 16 B)";
    case KVQ_E_UNSUPPORTED: return "kvquant_b200: unsupported configuration";
    default: break;
  }
  if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
  return "kvquant_b200: unknown error";
}

}  // extern "C"
