// common.cuh — shared infrastructure for libdinvk (sm_90a).
//
// Two build modes:
//   * nvcc (the product): real CUDA kernels launched on the caller's stream.
//   * DINVK_EMUL (tests/emul only, never shipped, never loaded by the package): the same SIMT
//     kernel sources are compiled by g++ against tests/emul/cuda_emul.h, which runs one block at a
//     time on host threads.  It exists so that kernel index math can be checked in the GPU-less
//     authoring container; it is test infrastructure like oracle/.
#pragma once

#include <cstdint>
#include <cstddef>
#include <cstdio>
#include <cstdarg>
#include <cmath>
#include <algorithm>
#include <utility>

#include "../../include/dinvk.h"

#ifdef DINVK_EMUL
#include "cuda_emul.h"
#else
#include <cuda_runtime.h>
#endif

// dynamic shared memory, usable from both build modes
#ifdef DINVK_EMUL
#define DINVK_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(::emul::dyn_smem())
#else
#define DINVK_DYN_SMEM(type, name)                                      \
  extern __shared__ __align__(16) unsigned char dinvk_dyn_smem_raw[];   \
  type* name = reinterpret_cast<type*>(dinvk_dyn_smem_raw)
#endif

namespace dinvk {

// ---- error plumbing -------------------------------------------------------------------------
char* err_buf();                 // thread-local, 512 bytes
int set_error(int code, const char* fmt, ...);
void count_launch();

// number of SMs the grids are sized against (H100 SXM: 132); queried once on the real device
int sm_count();

#define DINVK_CHECK_ARG(cond, ...)                                  \
  do {                                                              \
    if (!(cond)) return ::dinvk::set_error(DINVK_EINVAL, __VA_ARGS__); \
  } while (0)

#ifdef DINVK_EMUL
#define DINVK_LAUNCH(kernel, grid, block, smem, stream, ...)                      \
  do {                                                                            \
    ::dinvk::count_launch();                                                      \
    ::emul::launch((grid), (block), (size_t)(smem), [&]() { kernel(__VA_ARGS__); }); \
  } while (0)
#define DINVK_POST_LAUNCH() (0)
#else
#define DINVK_LAUNCH(kernel, grid, block, smem, stream, ...)                      \
  do {                                                                            \
    ::dinvk::count_launch();                                                      \
    kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);     \
  } while (0)
#define DINVK_POST_LAUNCH()                                                                   \
  ([]() -> int {                                                                              \
    cudaError_t e__ = cudaPeekAtLastError();                                                  \
    if (e__ != cudaSuccess) {                                                                 \
      (void)cudaGetLastError();                                                               \
      return ::dinvk::set_error(DINVK_ECUDA, "CUDA launch error: %s", cudaGetErrorString(e__)); \
    }                                                                                         \
    return 0;                                                                                 \
  }())
#endif

// opt-in to >48 KB dynamic shared memory (no-op under emulation).  The attribute belongs to the kernel on the current device,
// so it is raised once per (kernel, device), and again only when a launch needs more than was set.
int raise_smem_limit(const void* kernel, size_t bytes);
template <typename K>
inline int allow_smem(K kernel, size_t bytes) {
#ifndef DINVK_EMUL
  if (bytes > 48 * 1024) return raise_smem_limit(reinterpret_cast<const void*>(kernel), bytes);
#else
  (void)kernel; (void)bytes;
#endif
  return 0;
}

#ifndef DINVK_EMUL
// persistent kernels: min(work_items, SMs) CTAs, each looping over work items
template <typename... KArgs, typename... Args>
inline int launch_persistent(void (*kernel)(KArgs...), int threads, int smem, long long work_items, void* stream, Args&&... args) {
  int rc;
  if ((rc = allow_smem(kernel, smem))) return rc;
  const int grid = (int)std::min<long long>(work_items, sm_count());
  count_launch();
  kernel<<<grid, threads, smem, (cudaStream_t)stream>>>(std::forward<Args>(args)...);
  return DINVK_POST_LAUNCH();
}
#endif

// ---- tiny complex helpers -------------------------------------------------------------------
__host__ __device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__host__ __device__ __forceinline__ float2 cmul_conj(float2 a, float2 b) {  // a * conj(b)
  return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
__host__ __device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__host__ __device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__host__ __device__ __forceinline__ float2 cconj(float2 a) { return make_float2(a.x, -a.y); }

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// true if the product of the (non-negative) factors stays below 2^62: element / byte offsets of the tensor fit int64
inline bool product_fits(long long acc) { return acc >= 0; }
template <class... T>
inline bool product_fits(long long acc, long long f, T... rest) {
  return acc >= 0 && f >= 0 && (f == 0 || acc <= (1LL << 62) / f) && product_fits(acc * f, rest...);
}

}  // namespace dinvk
