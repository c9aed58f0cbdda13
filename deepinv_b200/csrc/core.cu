// core.cu — error reporting, launch counter, device query for libdinvk.
#include "common.cuh"

#include <atomic>

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

}  // namespace dinvk

extern "C" int dinvk_version(void) { return DINVK_VERSION; }
extern "C" const char* dinvk_last_error(void) { return dinvk::err_buf(); }
extern "C" uint64_t dinvk_launch_count(void) { return dinvk::g_launches.load(); }
