// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (see tma_util.h).
#include "tma_util.h"
#include "launch.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <map>
#include <mutex>
#include <set>
#include <utility>

#include "gemm_tc.h"

namespace lwb {

int& pdl_enabled() {
  static int v = 1;
  return v;
}

int ensure_max_dyn_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  std::lock_guard<std::mutex> lk(mu);
  if (done.count({kernel, dev})) return 0;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return static_cast<int>(e);
  done.insert({kernel, dev});
  return 0;
}

int current_device_sms() {
  static std::mutex mu;
  static std::map<int, int> sms;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  std::lock_guard<std::mutex> lk(mu);
  auto it = sms.find(dev);
  if (it != sms.end()) return it->second;
  int v = 0;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
  sms[dev] = v;
  return v;
}


typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled encode_fn() {
  static PFN_tmapEncodeTiled fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }();
  return fn;
}

int tma_encode(CUtensorMap* tm, int dtype, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, int swizzle_bytes, std::string* err) {
  PFN_tmapEncodeTiled fn = encode_fn();
  if (!fn) {
    *err = "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)";
    return -1;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUtensorMapSwizzle swz = swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMapDataType dt = dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                 : (dtype == DT_E4M3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  CUresult r = fn(tm, dt,
                  static_cast<cuuint32_t>(rank), const_cast<void*>(base), dims, strides_bytes, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (CUresult %d, rank %d, dim0 %llu, stride1 %llu, box0 %u)",
             static_cast<int>(r), rank, (unsigned long long)dims[0],
             (unsigned long long)(rank > 1 ? strides_bytes[0] : 0), box[0]);
    *err = buf;
    return -1;
  }
  return 0;
}

}  // namespace lwb
