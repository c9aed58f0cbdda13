// core.cu — error reporting, launch counter, device query, tensor-map encoder and shared-memory opt-in for libdinvk.
#include "common.cuh"
#include "tma_tile.cuh"

#include <atomic>
#include <map>
#include <mutex>

namespace dinvk {

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int sm_count() {
#ifdef DINVK_EMUL
  return 4;
#else
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;  // H100 SXM
    n = v;
  }
  return n;
#endif
}

#ifndef DINVK_EMUL
int raise_smem_limit(const void* kernel, size_t bytes) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> limit;  // (kernel, device) -> bytes set
  std::lock_guard<std::mutex> lock(mu);
  size_t& cur = limit[{kernel, dev}];
  if (bytes <= cur) return DINVK_OK;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e));
  cur = bytes;
  return DINVK_OK;
}

int encode_tiled(CUtensorMap* m, CUtensorMapDataType type, int rank, const void* ptr, const uint64_t* dims, const uint64_t* byte_strides,
                 const uint32_t* box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* what) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeTiledFn enc = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<EncodeTiledFn>(p);
  });
  if (!enc) return what ? set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable") : DINVK_ECUDA;
  const cuuint32_t elem_strides[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, type, (cuuint32_t)rank, const_cast<void*>(ptr), dims, byte_strides, box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return what ? set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r) : DINVK_ECUDA;
  return DINVK_OK;
}
#endif

}  // namespace dinvk

extern "C" int dinvk_version(void) { return DINVK_VERSION; }
extern "C" const char* dinvk_last_error(void) { return dinvk::err_buf(); }
extern "C" uint64_t dinvk_launch_count(void) { return dinvk::g_launches.load(); }
