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

// opt-in to >48 KB dynamic shared memory (no-op under emulation)
template <typename K>
inline int allow_smem(K kernel, size_t bytes) {
#ifndef DINVK_EMUL
  if (bytes > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e));
  }
#else
  (void)kernel; (void)bytes;
#endif
  return 0;
}

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

// number of SMs the grids are sized against (H100 SXM: 132); queried once on the real device
int sm_count();

}  // namespace dinvk
