// tma_tile.cuh — one TMA tensor-map load of an image tile (+ halo) into shared memory, out-of-range elements zero-filled by
// the copy engine: the staging step of the Radon and Blur kernels (north star: "TMA staging into shared memory").
// Host: a 3-D map (W, H, N) over a stack of fp32 images with a (box_w, box_h, 1) box; device: mbarrier + cp.async.bulk.tensor.3d
// (SASS: UTMALDG).  Requirements checked by the callers: 16-byte aligned base and row pitch (W % 4 == 0), box_w * 4 a multiple
// of 16, both box extents <= 256, 128-byte aligned shared-memory destination.
#pragma once
#ifndef DINVK_EMUL
#include <cuda.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace dinvk {

// The one tiled tensor-map encoder of the library (cuTensorMapEncodeTiled, resolved from the driver on first use): dims[0] is
// the contiguous axis, byte_strides holds the rank - 1 outer strides, unit element strides, no interleave, out-of-range
// elements read as zero.  Returns DINVK_OK, or DINVK_ECUDA with an error message naming `what` (no message when `what` is null).
int encode_tiled(CUtensorMap* m, CUtensorMapDataType type, int rank, const void* ptr, const uint64_t* dims, const uint64_t* byte_strides,
                 const uint32_t* box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2, const char* what);

namespace tt {

typedef CUtensorMap TileMap;

// true when the geometry can be expressed as a tensor map and the map was built (false: the caller stages cooperatively)
static inline bool make_map_f32(TileMap* m, const void* ptr, int W, int H, int N, int box_w, int box_h) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (W & 3) || (box_w & 3) || box_w > 256 || box_h > 256 || box_w < 1 || box_h < 1) return false;
  const uint64_t dims[3] = {(uint64_t)W, (uint64_t)H, (uint64_t)N};
  const uint64_t strides[2] = {(uint64_t)W * 4, (uint64_t)W * H * 4};
  const uint32_t box[3] = {(uint32_t)box_w, (uint32_t)box_h, 1};
  return encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, nullptr) == DINVK_OK;
}

__device__ __forceinline__ void tma_load_3d(void* smem, const TileMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   tc::smem_u32(smem)),
               "l"(reinterpret_cast<uint64_t>(m)), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

// whole-CTA helper: thread 0 arms the barrier and issues the box load; every thread returns when the tile has landed.
// `bar` is a shared 8-byte word used once per kernel (phase 0).
__device__ __forceinline__ void stage_tile(void* smem, const TileMap* m, uint64_t* bar, int x, int y, int n, uint32_t bytes) {
  if (threadIdx.x == 0) {
    tc::mbar_init(bar, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    tc::mbar_arrive_expect_tx(bar, bytes);
    tma_load_3d(smem, m, bar, x, y, n);
  }
  tc::mbar_wait(bar, 0);
}

}  // namespace tt
}  // namespace dinvk
#else
namespace dinvk {
namespace tt {
struct TileMap { int unused; };  // host emulation: the cooperative staging loop is used
}
}
#ifndef __grid_constant__
#define __grid_constant__
#endif
#endif
