// conv_tc.cu — bf16 tensor-core convolutions for the denoisers: wgmma implicit GEMM fed by TMA.
//
// Replaces the cuDNN/ATen calls behind deepinv/models/drunet.py:200-210 and dncnn.py:116-131 on the
// throughput path (fp32 parity path: conv_simt.cu).  Activations are NHWC bf16, weights (Cout, taps*Cin)
// bf16 K-major.  The GEMM view of a 3x3 convolution: M = output pixels, N = output channels,
// K = 9 taps x Cin; there is no im2col buffer — for each tap the A operand is the same NHWC tensor read
// through a 4-D TMA box shifted by (dx, dy); out-of-range coordinates are zero-filled by TMA, which IS the
// zero padding of the convolution.
//
// Kernel structure (one persistent CTA per SM):
//   warpgroups 0-1: consumers — warpgroup g issues wgmma (M=64, N=BN, K=16) for GEMM rows [64g, 64g+64) of the
//                   128-pixel tile, accumulates in registers (fp32) and runs the epilogue from its registers:
//                   + residual(s), ReLU, bf16 pack, NHWC stores, or fp32 NCHW stores for the network tail.
//   last warp     : TMA producer — per (tap, 64-channel block): one 4-D box (64 ch x 16 x x 8 y) of activations
//                   = 128 pixels x 128 B, and one 2-D box (64 k x BN rows) of weights, 128-byte swizzled,
//                   into an mbarrier-guarded ring of shared-memory stages.  While the consumers run an epilogue the
//                   producer already fills the ring for the next tile.
#include "common.cuh"
#include "tc_ptx.cuh"

#include <cstdlib>
#include <mutex>

namespace dinvk {

using bf16 = __nv_bfloat16;

constexpr int TC_TX = 16, TC_TY = 8;            // pixel tile: 16 x 8 = 128 GEMM rows
constexpr int TC_KB = 64;                        // K block: 64 bf16 = 128 B = one swizzle row
constexpr int TC_A_BYTES = 128 * TC_KB * 2;      // 16 KB
constexpr int TC_WG_ROWS = 64 * 128 >> 4;        // descriptor offset of GEMM row 64 (64 rows of 128 B, in 16-byte units)
constexpr int TC_THREADS = 2 * 128 + 32;         // two consumer warpgroups + the TMA producer warp

struct TcMaps {
  CUtensorMap a[4];  // activation views (3x3 and transposed-up: one; strided 2x2 down: one per tap)
  CUtensorMap b;     // weights
};

struct ConvTcParams {
  int B, H, W, Cin, Cout;       // H, W: pixel grid the GEMM rows tile (3x3: image; down: OUTPUT grid; up: INPUT grid)
                                // Cout = number of output channels actually stored
  int ntaps, kc_per_tap;
  int dx[9], dy[9], amap[9];    // per tap: box shift and which activation view to read
  int mode;                     // 0: NHWC bf16 same grid; 1: fp32 NCHW tail; 2: 2x up-scatter (GEMM column = tap*Cout + co)
  int tiles_x, tiles_y, n_tiles;
  int relu;
  const bf16* res;
  const bf16* res2;
  bf16* out;        // NHWC bf16 (B,H,W,Cout) or null
  float* out_f32;   // NCHW fp32 (B,Cout,H,W) or null (tail)
  const float* add_f32;  // optional NCHW fp32 term added in tail mode (DnCNN's "+ x")
  const float* bias;     // optional fp32 bias per output channel (DnCNN), added before the activation
};

template <int BN>
struct TcCfg {
  static constexpr int B_BYTES = BN * TC_KB * 2;
  static constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
  static constexpr int STAGES = BN >= 128 ? 6 : 8;
  static constexpr int SMEM = STAGES * STAGE_BYTES + 1024;  // + alignment slack
  static_assert(SMEM <= 227 * 1024, "shared memory budget");
};

template <int BN>
__device__ __forceinline__ void mma_bf16(float* d, uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi, uint32_t accumulate) {
  if constexpr (BN == 16) tc::wgmma_bf16_n16(d, a_lo, a_hi, b_lo, b_hi, accumulate);
  else if constexpr (BN == 64) tc::wgmma_bf16_n64(d, a_lo, a_hi, b_lo, b_hi, accumulate);
  else tc::wgmma_bf16_n128(d, a_lo, a_hi, b_lo, b_hi, accumulate);
}

// one warp's share of a consumed pipeline stage: the stage's `empty` barrier counts one arrival per consumer warp
__device__ __forceinline__ void release_stage(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) tc::mbar_arrive(bar);
}

__device__ __forceinline__ void named_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// epilogue of one m64 x BN accumulator fragment (see tc_ptx.cuh for the register layout): the caller maps the thread's two
// rows to pixels (y[r], x[r]); n0 = first GEMM column of the N tile
template <int BN>
__device__ __forceinline__ void epilogue_bf16(const ConvTcParams& P, const float* acc, int b, const int (&y)[2], const int (&x)[2], int n0) {
  const int q = threadIdx.x & 3;
  const int ncols = P.mode == 2 ? 4 * P.Cout : P.Cout;
  if (n0 >= ncols) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!(y[r] < P.H && x[r] < P.W)) continue;
    const long long pix = ((long long)b * P.H + y[r]) * P.W + x[r];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * q;
      float v0 = acc[4 * j + 2 * r], v1 = acc[4 * j + 2 * r + 1];
      if (P.bias) {
        v0 += (n < P.Cout) ? __ldg(P.bias + n) : 0.f;
        v1 += (n + 1 < P.Cout) ? __ldg(P.bias + n + 1) : 0.f;
      }
      if (P.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (P.out_f32) {
        // network tail: fp32 NCHW, only the real channels
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (n + e < P.Cout) {
            const long long o = (((long long)b * P.Cout + n + e) * P.H + y[r]) * P.W + x[r];
            float val = e ? v1 : v0;
            if (P.add_f32) val += __ldg(P.add_f32 + o);
            P.out_f32[o] = val;
          }
        }
      } else {
        long long o = pix * P.Cout + n;
        if (P.mode == 2) {  // transposed 2x2 stride-2: this N tile belongs to one (dy,dx) tap
          const int tap = n0 / P.Cout;
          o = (((long long)b * (2 * P.H) + 2 * y[r] + (tap >> 1)) * (2LL * P.W) + 2 * x[r] + (tap & 1)) * P.Cout + (n - tap * P.Cout);
        }
        if (P.res) { const float2 f = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(P.res + o))); v0 += f.x; v1 += f.y; }
        if (P.res2) { const float2 f = __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(P.res2 + o))); v0 += f.x; v1 += f.y; }
        *reinterpret_cast<__nv_bfloat162*>(P.out + o) = __floats2bfloat162_rn(v0, v1);
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ TcMaps M, const ConvTcParams P) {
  using Cfg = TcCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[Cfg::STAGES];
  __shared__ __align__(8) uint64_t empty_bar[Cfg::STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pixel_tiles = P.B * P.tiles_y * P.tiles_x;
  const int total_tiles = pixel_tiles * P.n_tiles;
  const int nk = P.ntaps * P.kc_per_tap;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&M.a[0]);
    tc::prefetch_tmap(&M.b);
    for (int s = 0; s < Cfg::STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 8); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t / pixel_tiles, pt = t - nt * pixel_tiles;
        const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
        const int y0 = (r / P.tiles_x) * TC_TY, x0 = (r % P.tiles_x) * TC_TX;
        for (int kb = 0; kb < nk; ++kb) {
          const int tap = kb / P.kc_per_tap, kc = kb - tap * P.kc_per_tap;
          tc::mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + TC_A_BYTES;
          tc::mbar_arrive_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
          tc::tma_load_4d(sa, &M.a[P.amap[tap]], &full_bar[s], kc * TC_KB, x0 + P.dx[tap], y0 + P.dy[tap], b);
          tc::tma_load_2d(sb, &M.b, &full_bar[s], tap * P.Cin + kc * TC_KB, nt * BN);
          if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma main loop + epilogue =====================
    // The group of stage kb is committed before the group of stage kb - 1 is waited for, so the tensor core always has
    // the next 4 MMAs queued; a stage goes back to the producer once the group that read it has completed.
    const int wg = warp >> 2;
    constexpr uint32_t HI = tc::desc_hi_sw128(1024);
    const uint32_t smem_lo = tc::smem_u32(smem) >> 4;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int nt = t / pixel_tiles, pt = t - nt * pixel_tiles;
      const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
      const int y0 = (r / P.tiles_x) * TC_TY, x0 = (r % P.tiles_x) * TC_TX;
      int pend = -1;
      for (int kb = 0; kb < nk; ++kb) {
        tc::mbar_wait(&full_bar[s], ph);
        const uint32_t a_lo = smem_lo + static_cast<uint32_t>(s) * (Cfg::STAGE_BYTES >> 4) + wg * TC_WG_ROWS;
        const uint32_t b_lo = smem_lo + static_cast<uint32_t>(s) * (Cfg::STAGE_BYTES >> 4) + (TC_A_BYTES >> 4);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) mma_bf16<BN>(acc, a_lo + 2 * k, HI, b_lo + 2 * k, HI, (kb | k) != 0 ? 1u : 0u);
        tc::wgmma_commit();
        tc::wgmma_wait<1>();
        if (pend >= 0) release_stage(&empty_bar[pend]);
        pend = s;
        if (++s == Cfg::STAGES) { s = 0; ph ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::reg_fence<BN / 2>(acc);
      if (pend >= 0) release_stage(&empty_bar[pend]);
      int y[2], x[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * rr;
        y[rr] = y0 + m / TC_TX; x[rr] = x0 + m % TC_TX;
      }
      epilogue_bf16<BN>(P, acc, b, y, x, nt * BN);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 3x3 convolution with HALO REUSE (64- and 128-channel layers).
//
// The per-tap kernel above re-reads every activation tile 9 times from L2.  Here one TMA box brings an (18 y) x (SLAB_X x)
// x 64-channel slab (the output tile plus its halo; a multiple of 8 positions per slab row keeps every 8-row group
// 1024-byte periodic) into shared memory ONCE per 64-channel block, and the nine taps are nine wgmma descriptors into that
// same slab: start address shifted by (ky*SLAB_X + kx) rows of 128 B, stride between 8-row groups = one slab row.  The
// 128-byte swizzle is a function of the shared-memory ADDRESS bits on both the TMA write and the wgmma read, so a start
// address that is not 1024-byte aligned needs no descriptor base offset.  L2->SM activation traffic drops about 4x.
// For 64->64 layers the whole weight tensor (9 x 64 x 64 bf16 = 72 KB) stays resident in shared memory for the lifetime
// of the CTA.
// ---------------------------------------------------------------------------------------------------------------
// MH x-halves per CTA tile: the tile is 8*MH x by 16 y output pixels.  Consumer warpgroup g owns the m64 block
// (x-half g / 2, y-half g % 2): 8 x 8 pixels, GEMM row m = 8 * (y - y-half start) + (x - x-half start).
// MH = 2 shares every weight tile between four warpgroups (256 pixels per B stage).
constexpr int HL_TY = 16;
template <int MH> struct HaloGeom {
  static constexpr int TX = 8 * MH;
  static constexpr int SLAB_X = TX + 8;              // >= TX + 2, multiple of 8 so that every slab row is 1024-byte periodic
  static constexpr int SLAB_Y = HL_TY + 2;
  static constexpr int SLAB_BYTES = SLAB_X * SLAB_Y * 128;
};

// AST: activation slabs in flight; BST: weight tiles in the ring (streamed mode).  BN = 16 is the network tail
// (64 -> Cout <= 16, fp32 NCHW output).
template <int BN, bool RESIDENT, int AST, int BST, int MH>
struct HaloCfg {
  using G = HaloGeom<MH>;
  static constexpr int B_TILE = BN * 128;
  static constexpr int A_STAGES = AST;
  static constexpr int B_STAGES = RESIDENT ? 9 : BST;
  static constexpr int SMEM = A_STAGES * G::SLAB_BYTES + B_STAGES * B_TILE + 1024;
  static_assert(SMEM <= 227 * 1024, "shared memory budget");
  static_assert(G::SLAB_BYTES % 1024 == 0, "slab stages must stay 1024-byte aligned");
  static constexpr int NWG = 2 * MH;                 // consumer warpgroups
  static constexpr int THREADS = 128 * NWG + 32;     // + the TMA producer warp
};

template <int BN, bool RESIDENT, int AST, int BST, int MH>
__global__ void __launch_bounds__((HaloCfg<BN, RESIDENT, AST, BST, MH>::THREADS), 1)
conv_tc_halo_kernel(const __grid_constant__ TcMaps M, const ConvTcParams P) {
  using Cfg = HaloCfg<BN, RESIDENT, AST, BST, MH>;
  using G = HaloGeom<MH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_b = smem + Cfg::A_STAGES * G::SLAB_BYTES;
  __shared__ __align__(8) uint64_t afull[Cfg::A_STAGES];
  __shared__ __align__(8) uint64_t aempty[Cfg::A_STAGES];
  __shared__ __align__(8) uint64_t bfull[Cfg::B_STAGES];
  __shared__ __align__(8) uint64_t bempty[Cfg::B_STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pixel_tiles = P.B * P.tiles_y * P.tiles_x;
  const int total_tiles = pixel_tiles * P.n_tiles;
  const int nkc = P.kc_per_tap;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&M.a[0]);
    tc::prefetch_tmap(&M.b);
    for (int s = 0; s < Cfg::A_STAGES; ++s) { tc::mbar_init(&afull[s], 1); tc::mbar_init(&aempty[s], 4 * Cfg::NWG); }
    for (int s = 0; s < Cfg::B_STAGES; ++s) { tc::mbar_init(&bfull[s], 1); tc::mbar_init(&bempty[s], 4 * Cfg::NWG); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 * Cfg::NWG) {
    if (lane == 0) {
      if (RESIDENT) {  // the whole 3x3 weight tensor, once
        for (int tap = 0; tap < 9; ++tap) {
          tc::mbar_arrive_expect_tx(&bfull[tap], Cfg::B_TILE);
          tc::tma_load_2d(smem_b + tap * Cfg::B_TILE, &M.b, &bfull[tap], tap * P.Cin, 0);
        }
      }
      int sa = 0; uint32_t pha = 0;
      int sb = 0; uint32_t phb = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t / pixel_tiles, pt = t - nt * pixel_tiles;
        const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
        const int y0 = (r / P.tiles_x) * HL_TY, x0 = (r % P.tiles_x) * G::TX;
        for (int kc = 0; kc < nkc; ++kc) {
          tc::mbar_wait(&aempty[sa], pha ^ 1);
          tc::mbar_arrive_expect_tx(&afull[sa], G::SLAB_BYTES);
          tc::tma_load_4d(smem + sa * G::SLAB_BYTES, &M.a[0], &afull[sa], kc * TC_KB, x0 - 1, y0 - 1, b);
          if (++sa == Cfg::A_STAGES) { sa = 0; pha ^= 1; }
          if (!RESIDENT) {
            for (int tap = 0; tap < 9; ++tap) {
              tc::mbar_wait(&bempty[sb], phb ^ 1);
              tc::mbar_arrive_expect_tx(&bfull[sb], Cfg::B_TILE);
              tc::tma_load_2d(smem_b + sb * Cfg::B_TILE, &M.b, &bfull[sb], tap * P.Cin + kc * TC_KB, nt * BN);
              if (++sb == Cfg::B_STAGES) { sb = 0; phb ^= 1; }
            }
          }
        }
      }
    }
  } else {
    const int wg = warp >> 2;
    const int half = wg >> 1, yh = wg & 1;
    constexpr uint32_t HI_A = tc::desc_hi_sw128(G::SLAB_X * 128);
    constexpr uint32_t HI_B = tc::desc_hi_sw128(1024);
    // this warpgroup's block starts at slab row 8 * yh, position 8 * half (128-byte rows = 8 descriptor units)
    const uint32_t slab_lo0 = (tc::smem_u32(smem) >> 4) + static_cast<uint32_t>((8 * yh * G::SLAB_X + 8 * half) * 8);
    const uint32_t bt_lo0 = tc::smem_u32(smem_b) >> 4;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int sa = 0; uint32_t pha = 0;
    int sb = 0; uint32_t phb = 0;
    if (RESIDENT) {
      for (int tap = 0; tap < 9; ++tap) tc::mbar_wait(&bfull[tap], 0);
    }
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int nt = t / pixel_tiles, pt = t - nt * pixel_tiles;
      const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
      const int y0 = (r / P.tiles_x) * HL_TY, x0 = (r % P.tiles_x) * G::TX;
      int pend_a = -1, pend_b = -1;  // stages read by the previous wgmma group: released once it has completed
      for (int kc = 0; kc < nkc; ++kc) {
        tc::mbar_wait(&afull[sa], pha);
        const uint32_t slab_lo = slab_lo0 + static_cast<uint32_t>(sa) * (G::SLAB_BYTES >> 4);
        if (RESIDENT) {
          tc::wgmma_fence();
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const uint32_t a_lo = slab_lo + static_cast<uint32_t>(((tap / 3) * G::SLAB_X + (tap % 3)) * 8);
            const uint32_t b_lo = bt_lo0 + static_cast<uint32_t>(tap * (Cfg::B_TILE >> 4));
#pragma unroll
            for (int k = 0; k < 4; ++k) mma_bf16<BN>(acc, a_lo + 2 * k, HI_A, b_lo + 2 * k, HI_B, (kc | tap | k) != 0 ? 1u : 0u);
          }
          tc::wgmma_commit();
          tc::wgmma_wait<1>();
          if (pend_a >= 0) release_stage(&aempty[pend_a]);
          pend_a = sa;
        } else {
#pragma unroll 1
          for (int tap = 0; tap < 9; ++tap) {
            tc::mbar_wait(&bfull[sb], phb);
            const uint32_t a_lo = slab_lo + static_cast<uint32_t>(((tap / 3) * G::SLAB_X + (tap % 3)) * 8);
            const uint32_t b_lo = bt_lo0 + static_cast<uint32_t>(sb) * (Cfg::B_TILE >> 4);
            tc::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) mma_bf16<BN>(acc, a_lo + 2 * k, HI_A, b_lo + 2 * k, HI_B, (kc | tap | k) != 0 ? 1u : 0u);
            tc::wgmma_commit();
            tc::wgmma_wait<1>();
            if (pend_b >= 0) release_stage(&bempty[pend_b]);
            if (pend_a >= 0) release_stage(&aempty[pend_a]);
            pend_b = sb;
            pend_a = tap == 8 ? sa : -1;
            if (++sb == Cfg::B_STAGES) { sb = 0; phb ^= 1; }
          }
        }
        if (++sa == Cfg::A_STAGES) { sa = 0; pha ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::reg_fence<BN / 2>(acc);
      if (pend_b >= 0) release_stage(&bempty[pend_b]);
      if (pend_a >= 0) release_stage(&aempty[pend_a]);
      int y[2], x[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = 16 * (warp & 3) + (lane >> 2) + 8 * rr;
        y[rr] = y0 + 8 * yh + (m >> 3); x[rr] = x0 + 8 * half + (m & 7);
      }
      epilogue_bf16<BN>(P, acc, b, y, x, nt * BN);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Network HEAD: 3x3 convolution from a few-channel NCHW fp32 image (+ optional constant noise-level channel, DRUNet's
// sigma map) to 64 NHWC bf16 channels.  Going through the generic kernel means padding 3 channels to 64 (a large
// converter write and 9 taps x 64 channels of zeros through L2 and the tensor pipe).
// Here the im2col row of a pixel (K = 9 taps x CT channels <= 64, k = tap*CT + c) is BUILT IN SHARED MEMORY by CUDA
// threads straight from the fp32 input, in the 128-byte-swizzled K-major layout the wgmma descriptor expects
// (16-byte chunk j of row m lives at chunk j ^ (m & 7)), so the whole layer is one K=64 GEMM step per 128-pixel tile
// and the only real traffic is the output write.
//   warpgroup g (of 2) owns every other tile: its 128 threads build the tile's 128 rows (one pixel each) in A stage g,
//   issue 2 x 4 wgmma (M=64, N=64, K=16) and store the two m64 accumulators.
// ---------------------------------------------------------------------------------------------------------------
struct HeadParams {
  const float* x;          // (B, C, H, W) fp32
  const bf16* w;           // (64, 64) bf16, k = tap*CT + c, zero padded
  const float* bias;       // optional (64)
  bf16* out;               // (B, H, W, 64)
  int B, C, H, W;
  float fill_scalar;
  const float* fill_batch;
  int has_fill;
  int relu;
  int tiles_x, tiles_y;
};
constexpr int HD_TX = 32, HD_TY = 4;
constexpr int HD_THREADS = 2 * 128;
constexpr int HD_SMEM = 2 * TC_A_BYTES + 64 * 128 + 1024;

template <int CT>
__global__ void __launch_bounds__(HD_THREADS, 1) conv_head_kernel(const HeadParams P) {
  constexpr int KREAL = 9 * CT;
  constexpr int NCH = (KREAL + 7) / 8;  // 16-byte chunks rewritten for every tile
  static_assert(KREAL <= 64, "head: 9 * channels must fit one 64-wide K block");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_b = smem + 2 * TC_A_BYTES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = P.B * P.tiles_y * P.tiles_x;

  // zero both A stages once (chunks >= NCH are never written again), stage the weights with the same swizzle
  for (int i = threadIdx.x; i < 2 * TC_A_BYTES / 16; i += HD_THREADS) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 64 * 8; i += HD_THREADS) {
    const int n = i >> 3, j = i & 7;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(P.w) + i);
    *reinterpret_cast<uint4*>(smem_b + n * 128 + ((j ^ (n & 7)) << 4)) = v;
  }
  tc::fence_proxy_async();
  __syncthreads();

  // The 9*CT input values of a pixel are fetched with UNCONDITIONAL loads from clamped coordinates (then masked), one
  // tile ahead of their use: all loads of a tile are independent and in flight while the previous tile is converted,
  // stored and multiplied.
  const int group = warp >> 2;
  const int m = (warp & 3) * 32 + lane;  // GEMM row = (warp&3) tile row, lane = x
  uint8_t* row = smem + group * TC_A_BYTES + m * 128;
  const int tiles_per_img = P.tiles_y * P.tiles_x;
  auto gather = [&](int t, float (&v)[9 * CT]) {
    const int b = t / tiles_per_img, r = t - b * tiles_per_img;
    const int y = (r / P.tiles_x) * HD_TY + (warp & 3), x = (r % P.tiles_x) * HD_TX + lane;
    const float fillv = P.has_fill ? (P.fill_batch ? __ldg(P.fill_batch + b) : P.fill_scalar) : 0.f;
    const float* img = P.x + (long long)b * P.C * P.H * P.W;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
      const bool inb = (yy >= 0) && (yy < P.H) && (xx >= 0) && (xx < P.W);
      const int yc = min(max(yy, 0), P.H - 1), xc = min(max(xx, 0), P.W - 1);
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        const int cc = min(c, P.C - 1);
        const float val = __ldg(img + ((long long)cc * P.H + yc) * P.W + xc);
        v[tap * CT + c] = inb ? ((c < P.C) ? val : fillv) : 0.f;  // a select, not a branch: the load above is unconditional
      }
    }
  };
  constexpr uint32_t HI = tc::desc_hi_sw128(1024);
  const uint32_t a_lo = (tc::smem_u32(smem) >> 4) + static_cast<uint32_t>(group) * (TC_A_BYTES >> 4);
  const uint32_t b_lo = tc::smem_u32(smem_b) >> 4;
  float acc[2][32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
  const int stride2 = 2 * gridDim.x;
  int t = blockIdx.x + group * gridDim.x;
  float cur[9 * CT];
  if (t < total_tiles) gather(t, cur);
  for (; t < total_tiles; t += stride2) {
    float nxt[9 * CT];
    const bool more = t + stride2 < total_tiles;
    if (more) gather(t + stride2, nxt);
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k0 = j * 8 + 2 * e;
        h[e] = __floats2bfloat162_rn(k0 < KREAL ? cur[k0] : 0.f, k0 + 1 < KREAL ? cur[k0 + 1] : 0.f);
      }
      *reinterpret_cast<uint4*>(row + ((j ^ (m & 7)) << 4)) = u;
    }
    tc::fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
    named_sync(1 + group, 128);
    tc::wgmma_fence();
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int k = 0; k < 4; ++k) tc::wgmma_bf16_n64(acc[hh], a_lo + hh * TC_WG_ROWS + 2 * k, HI, b_lo + 2 * k, HI, k != 0 ? 1u : 0u);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence<32>(acc[0]);
    tc::reg_fence<32>(acc[1]);
    named_sync(1 + group, 128);  // every warp's reads of the A stage are complete before it is rewritten
    const int b = t / tiles_per_img, r = t - b * tiles_per_img;
    const int y0 = (r / P.tiles_x) * HD_TY, x0 = (r % P.tiles_x) * HD_TX;
    const int q = lane & 3;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int mm = 64 * hh + 16 * (warp & 3) + (lane >> 2) + 8 * rr;
        const int y = y0 + mm / HD_TX, x = x0 + mm % HD_TX;
        if (y >= P.H || x >= P.W) continue;
        bf16* o = P.out + (((long long)b * P.H + y) * P.W + x) * 64;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * q;
          float v0 = acc[hh][4 * j + 2 * rr], v1 = acc[hh][4 * j + 2 * rr + 1];
          if (P.bias) { v0 += __ldg(P.bias + c); v1 += __ldg(P.bias + c + 1); }
          if (P.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          *reinterpret_cast<__nv_bfloat162*>(o + c) = __floats2bfloat162_rn(v0, v1);
        }
      }
    if (more) {
#pragma unroll
      for (int k = 0; k < 9 * CT; ++k) cur[k] = nxt[k];
    }
  }
}

// ---- layout converters ---------------------------------------------------------------------------------
// NCHW fp32 -> NHWC bf16 with channel padding; channel C is filled with the noise level (DRUNet's sigma map)
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const float* __restrict__ in, bf16* __restrict__ out, int C, int H, int W,
                                                           int Cpad, float fill_scalar, const float* __restrict__ fill_batch,
                                                           int has_fill, long long npix) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long HW = (long long)H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += stride) {
    const long long b = p / HW, hw = p - b * HW;
    bf16* o = out + p * Cpad;
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float f[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int c = c0 + 2 * e + k;
          float val = 0.f;
          if (c < C) val = __ldg(in + (b * C + c) * HW + hw);
          else if (c == C && has_fill) val = fill_batch ? __ldg(fill_batch + b) : fill_scalar;
          f[k] = val;
        }
        h[e] = __floats2bfloat162_rn(f[0], f[1]);
      }
      *reinterpret_cast<uint4*>(o + c0) = u;
    }
  }
}

__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const bf16* __restrict__ in, const float* __restrict__ add,
                                                           float* __restrict__ out, int C, int H, int W, int Cpad, long long npix) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long HW = (long long)H * W;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += stride) {
    const long long b = p / HW, hw = p - b * HW;
    for (int c = 0; c < C; ++c) {
      const long long o = (b * C + c) * HW + hw;
      float v = __bfloat162float(in[p * Cpad + c]);
      if (add) v += __ldg(add + o);
      out[o] = v;
    }
  }
}

// ---- 2x2 stride-2 down / transposed up (bf16 NHWC, CUDA cores; < 3 % of DRUNet's FLOPs) -----------------
// down: out[b,yo,xo,co] = sum_{dy,dx,c} w[co, (dy*2+dx)*Cin + c] * (x + xadd)[b, 2yo+dy, 2xo+dx, c]
// up  : out[b,2y+dy,2x+dx,co] = sum_c w[(dy*2+dx)*Cout + co, c] * (x + xadd)[b, y, x, c]
// one CTA: 32 GEMM rows x 64 GEMM columns, K staged through shared memory in chunks of 64
template <bool UP>
__global__ void __launch_bounds__(256) conv2x2_bf16_kernel(const bf16* __restrict__ x, const bf16* __restrict__ xadd,
                                                           const bf16* __restrict__ w, bf16* __restrict__ out, int B, int H, int W,
                                                           int Cin, int Cout) {
  constexpr int TM = 32, TN = 64, TK = 64;
  __shared__ float sA[TK][TM + 1];
  __shared__ float sW[TK][TN + 1];
  const int Ho = H / 2, Wo = W / 2;
  const long long M = UP ? (long long)B * H * W : (long long)B * Ho * Wo;
  const int N = UP ? 4 * Cout : Cout;
  const int K = UP ? Cin : 4 * Cin;
  const long long m0 = (long long)blockIdx.x * TM;
  const int n0 = blockIdx.y * TN;
  const int tid = threadIdx.x;
  const int tm = tid & 31, tn = tid >> 5;  // thread: row tm, columns tn*8 .. tn*8+7
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int k0 = 0; k0 < K; k0 += TK) {
    for (int idx = tid; idx < TM * TK; idx += 256) {
      const int mm = idx / TK, kk = idx - mm * TK;  // k fastest: contiguous channels
      const long long m = m0 + mm;
      const int k = k0 + kk;
      float v = 0.f;
      if (m < M && k < K) {
        long long o;
        if (UP) {
          o = m * Cin + k;
        } else {
          const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho);
          const long long bb = m / ((long long)Wo * Ho);
          const int tap = k / Cin, c = k - tap * Cin;
          o = ((bb * H + 2 * yo + (tap >> 1)) * W + 2 * xo + (tap & 1)) * Cin + c;
        }
        v = __bfloat162float(x[o]);
        if (xadd) v += __bfloat162float(xadd[o]);
      }
      sA[kk][mm] = v;
    }
    for (int idx = tid; idx < TN * TK; idx += 256) {
      const int nn = idx / TK, kk = idx - nn * TK;
      const int n = n0 + nn, k = k0 + kk;
      sW[kk][nn] = (n < N && k < K) ? __bfloat162float(w[(long long)n * K + k]) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < TK; ++kk) {
      const float a = sA[kk][tm];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(a, sW[kk][tn * 8 + i], acc[i]);
    }
    __syncthreads();
  }
  const long long m = m0 + tm;
  if (m < M) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int n = n0 + tn * 8 + i;
      if (n >= N) continue;
      long long o;
      if (UP) {
        const long long HWl = (long long)H * W;
        const long long bb = m / HWl, p = m - bb * HWl;
        const int y = (int)(p / W), xx = (int)(p - (long long)y * W);
        const int tap = n / Cout, co = n - tap * Cout;
        o = ((bb * (2 * H) + 2 * y + (tap >> 1)) * (2LL * W) + 2 * xx + (tap & 1)) * Cout + co;
      } else {
        o = m * Cout + n;
      }
      out[o] = __float2bfloat16(acc[i]);
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 4-D activation view (C, X, Y, B) with arbitrary element strides (bytes) — plain NHWC for 3x3 / up, a stride-2
// sub-lattice of the input for each tap of the 2x2 down-conv
static int make_act_map(CUtensorMap* m, const void* ptr, int B, int Y, int X, int C, long long sx, long long sy, long long sb) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)X, (cuuint64_t)Y, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)sx, (cuuint64_t)sy, (cuuint64_t)sb};
  cuuint32_t box[4] = {TC_KB, TC_TX, TC_TY, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(activations) failed: %d", (int)r);
  return 0;
}
static int make_w_map(CUtensorMap* m, const void* ptr, int K, int rows, int bn) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {TC_KB, (cuuint32_t)bn};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(weights) failed: %d", (int)r);
  return 0;
}

template <int BN>
static int launch_conv_tc(const TcMaps& M, const ConvTcParams& P, void* stream) {
  using Cfg = TcCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(conv_tc<%d>): %s", BN, cudaGetErrorString(e));
    attr_set = true;
  }
  const long long tiles = (long long)P.B * P.tiles_y * P.tiles_x * P.n_tiles;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  count_launch();
  conv_tc_kernel<BN><<<grid, TC_THREADS, Cfg::SMEM, (cudaStream_t)stream>>>(M, P);
  return DINVK_POST_LAUNCH();
}

static int make_slab_map(CUtensorMap* m, const void* ptr, int B, int H, int W, int C, int slab_x) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {TC_KB, (cuuint32_t)slab_x, HL_TY + 2, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(slab) failed: %d", (int)r);
  return 0;
}

template <int BN, bool RESIDENT, int AST, int BST, int MH>
static int launch_conv_halo(TcMaps& M, ConvTcParams& P, const void* x, void* stream) {
  using Cfg = HaloCfg<BN, RESIDENT, AST, BST, MH>;
  using G = HaloGeom<MH>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_halo_kernel<BN, RESIDENT, AST, BST, MH>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(conv_tc_halo<%d>): %s", BN, cudaGetErrorString(e));
    attr_set = true;
  }
  int rc;
  if ((rc = make_slab_map(&M.a[0], x, P.B, P.H, P.W, P.Cin, G::SLAB_X))) return rc;
  M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
  P.tiles_x = ceil_div(P.W, G::TX); P.tiles_y = ceil_div(P.H, HL_TY);
  const long long tiles = (long long)P.B * P.tiles_y * P.tiles_x * P.n_tiles;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  count_launch();
  conv_tc_halo_kernel<BN, RESIDENT, AST, BST, MH><<<grid, Cfg::THREADS, Cfg::SMEM, (cudaStream_t)stream>>>(M, P);
  return DINVK_POST_LAUNCH();
}

// halo mode (DINVK_CONV_HALO): 0 = off (per-tap kernel), 1 = on (default).
static int halo_mode() {
  static int mode = -1;
  if (mode < 0) {
    const char* e = getenv("DINVK_CONV_HALO");
    mode = e ? atoi(e) : 1;
  }
  return mode;
}

// N tile: at most 128 columns, so that a consumer warpgroup's m64 accumulator is at most 64 registers per thread
static int pick_bn(int rows) { return rows % 128 == 0 ? 128 : 64; }

static int dispatch_conv_tc(int bn, const TcMaps& M, const ConvTcParams& P, void* stream) {
  switch (bn) {
    case 16: return launch_conv_tc<16>(M, P, stream);
    case 64: return launch_conv_tc<64>(M, P, stream);
    default: return launch_conv_tc<128>(M, P, stream);
  }
}

static int conv3x3_tc(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                      float* out_f32, const float* add_f32, int B, int H, int W, int Cin, int Cout_real, int rows, int act, void* stream) {
  DINVK_CHECK_ARG(x && weight && (out || out_f32), "conv3x3_bf16: null pointer");
  DINVK_CHECK_ARG(B >= 0 && H >= 1 && W >= 1, "conv3x3_bf16: bad shape");
  DINVK_CHECK_ARG(Cin % 64 == 0 && Cin >= 64, "conv3x3_bf16: Cin=%d must be a multiple of 64", Cin);
  DINVK_CHECK_ARG(out_f32 || (Cout_real % 64 == 0), "conv3x3_bf16: Cout=%d must be a multiple of 64", Cout_real);
  if (B == 0) return DINVK_OK;
  const int bn = out_f32 ? 16 : pick_bn(rows);
  DINVK_CHECK_ARG(rows % bn == 0, "conv3x3_bf16: weight rows %d not a multiple of the N tile %d", rows, bn);
  TcMaps M;
  int rc;
  // slab + halo kernel (activations read once per 64-channel block instead of once per tap):
  //   64 -> 64 and the 64 -> (<=16) tail with the weights resident in shared memory; >= 128 output channels with streamed
  //   weights.  64-channel layers use 16x16-pixel CTA tiles (four m64 blocks share every weight tile), the streamed layers
  //   8x16-pixel tiles (two m64 blocks of up to 64 accumulator registers per thread).
  const bool halo_tail = out_f32 && Cin == 64 && rows == 16 && !getenv("DINVK_NO_HALO_TAIL");
  const bool halo_body = !out_f32 && ((rows == 64 && Cin == 64) || bn == 128);
  if (halo_mode() != 0 && (halo_tail || halo_body)) {
    if ((rc = make_w_map(&M.b, weight, 9 * Cin, rows, bn))) return rc;
    ConvTcParams P;
    P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout_real;
    P.ntaps = 9; P.kc_per_tap = Cin / TC_KB;
    for (int t = 0; t < 9; ++t) { P.dx[t] = t % 3 - 1; P.dy[t] = t / 3 - 1; P.amap[t] = 0; }
    P.mode = out_f32 ? 1 : 0;
    P.tiles_x = 0; P.tiles_y = 0; P.n_tiles = rows / bn;  // tiles_x/y: set by the launcher from the kernel's tile geometry
    P.relu = act; P.res = (const bf16*)res; P.res2 = (const bf16*)res2; P.out = (bf16*)out; P.out_f32 = out_f32; P.add_f32 = add_f32; P.bias = bias;
    if (halo_tail) return launch_conv_halo<16, true, 4, 0, 1>(M, P, x, stream);
    if (bn == 64) return launch_conv_halo<64, true, 2, 0, 2>(M, P, x, stream);
    return launch_conv_halo<128, false, 2, 8, 1>(M, P, x, stream);
  }
  if ((rc = make_act_map(&M.a[0], x, B, H, W, Cin, (long long)Cin * 2, (long long)W * Cin * 2, (long long)H * W * Cin * 2))) return rc;
  M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
  if ((rc = make_w_map(&M.b, weight, 9 * Cin, rows, bn))) return rc;
  ConvTcParams P;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout_real;
  P.ntaps = 9; P.kc_per_tap = Cin / TC_KB;
  for (int t = 0; t < 9; ++t) { P.dx[t] = t % 3 - 1; P.dy[t] = t / 3 - 1; P.amap[t] = 0; }
  P.mode = out_f32 ? 1 : 0;
  P.tiles_x = ceil_div(W, TC_TX); P.tiles_y = ceil_div(H, TC_TY); P.n_tiles = rows / bn;
  P.relu = act; P.res = (const bf16*)res; P.res2 = (const bf16*)res2; P.out = (bf16*)out; P.out_f32 = out_f32; P.add_f32 = add_f32; P.bias = bias;
  return dispatch_conv_tc(bn, M, P, stream);
}

// 2x2 stride-2 convolution as a 4-tap implicit GEMM: tap (dy,dx) reads the stride-2 sub-lattice of the input that
// starts at (dy,dx) through its own tensor map; GEMM rows tile the OUTPUT grid
static int conv2x2_down_tc(const void* x, const void* weight, void* out, int B, int H, int W, int Cin, int Cout, void* stream) {
  const int Ho = H / 2, Wo = W / 2;
  const int bn = pick_bn(Cout);
  TcMaps M;
  int rc;
  for (int t = 0; t < 4; ++t) {
    const char* base = static_cast<const char*>(x) + ((long long)(t >> 1) * W + (t & 1)) * Cin * 2;
    if ((rc = make_act_map(&M.a[t], base, B, Ho, Wo, Cin, 2LL * Cin * 2, 2LL * W * Cin * 2, (long long)H * W * Cin * 2))) return rc;
  }
  if ((rc = make_w_map(&M.b, weight, 4 * Cin, Cout, bn))) return rc;
  ConvTcParams P;
  P.B = B; P.H = Ho; P.W = Wo; P.Cin = Cin; P.Cout = Cout;
  P.ntaps = 4; P.kc_per_tap = Cin / TC_KB;
  for (int t = 0; t < 9; ++t) { P.dx[t] = 0; P.dy[t] = 0; P.amap[t] = t < 4 ? t : 0; }
  P.mode = 0;
  P.tiles_x = ceil_div(Wo, TC_TX); P.tiles_y = ceil_div(Ho, TC_TY); P.n_tiles = Cout / bn;
  P.relu = 0; P.res = nullptr; P.res2 = nullptr; P.out = (bf16*)out; P.out_f32 = nullptr; P.add_f32 = nullptr; P.bias = nullptr;
  return dispatch_conv_tc(bn, M, P, stream);
}

// transposed 2x2 stride-2 convolution as a 1-tap GEMM with N = 4*Cout (column = tap*Cout + co) and a scatter epilogue
static int conv2x2_up_tc(const void* x, const void* weight, void* out, int B, int H, int W, int Cin, int Cout, void* stream) {
  const int bn = pick_bn(Cout);  // an N tile never spans two taps
  TcMaps M;
  int rc;
  if ((rc = make_act_map(&M.a[0], x, B, H, W, Cin, (long long)Cin * 2, (long long)W * Cin * 2, (long long)H * W * Cin * 2))) return rc;
  M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
  if ((rc = make_w_map(&M.b, weight, Cin, 4 * Cout, bn))) return rc;
  ConvTcParams P;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout;
  P.ntaps = 1; P.kc_per_tap = Cin / TC_KB;
  for (int t = 0; t < 9; ++t) { P.dx[t] = 0; P.dy[t] = 0; P.amap[t] = 0; }
  P.mode = 2;
  P.tiles_x = ceil_div(W, TC_TX); P.tiles_y = ceil_div(H, TC_TY); P.n_tiles = 4 * Cout / bn;
  P.relu = 0; P.res = nullptr; P.res2 = nullptr; P.out = (bf16*)out; P.out_f32 = nullptr; P.add_f32 = nullptr; P.bias = nullptr;
  return dispatch_conv_tc(bn, M, P, stream);
}

}  // namespace dinvk

using namespace dinvk;

extern "C" int dinvk_conv3x3_bf16(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                                  int B, int H, int W, int Cin, int Cout, int act, void* stream) {
  return conv3x3_tc(x, weight, bias, res, res2, out, nullptr, nullptr, B, H, W, Cin, Cout, Cout, act, stream);
}

extern "C" int dinvk_conv3x3_bf16_tail(const void* x, const void* weight16, const float* bias, const float* add_nchw,
                                       float* out_nchw, int B, int H, int W, int Cin, int Cout, void* stream) {
  DINVK_CHECK_ARG(Cout >= 1 && Cout <= 16, "conv3x3_bf16_tail: Cout=%d must be <= 16", Cout);
  return conv3x3_tc(x, weight16, bias, nullptr, nullptr, nullptr, out_nchw, add_nchw, B, H, W, Cin, Cout, 16, 0, stream);
}

template <int CT>
static int launch_head(const HeadParams& P, void* stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_head_kernel<CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, HD_SMEM);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(conv_head<%d>): %s", CT, cudaGetErrorString(e));
    attr_set = true;
  }
  const long long tiles = (long long)P.B * P.tiles_y * P.tiles_x;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  count_launch();
  conv_head_kernel<CT><<<grid, HD_THREADS, HD_SMEM, (cudaStream_t)stream>>>(P);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_conv3x3_head_bf16(const float* x_nchw, const void* weight64, const float* bias, void* out_nhwc, int B, int C, int H,
                                       int W, float fill_scalar, const float* fill_batch, int has_fill, int act, void* stream) {
  DINVK_CHECK_ARG(x_nchw && weight64 && out_nhwc && B >= 0 && C >= 1 && H >= 1 && W >= 1, "conv3x3_head_bf16: bad arguments");
  const int CT = C + (has_fill ? 1 : 0);
  DINVK_CHECK_ARG(CT >= 1 && CT <= 4, "conv3x3_head_bf16: %d input channels (incl. noise map) not in 1..4", CT);
  if (B == 0) return DINVK_OK;
  HeadParams P;
  P.x = x_nchw; P.w = (const bf16*)weight64; P.bias = bias; P.out = (bf16*)out_nhwc;
  P.B = B; P.C = C; P.H = H; P.W = W;
  P.fill_scalar = fill_scalar; P.fill_batch = fill_batch; P.has_fill = has_fill; P.relu = act;
  P.tiles_x = ceil_div(W, HD_TX); P.tiles_y = ceil_div(H, HD_TY);
  switch (CT) {
    case 1: return launch_head<1>(P, stream);
    case 2: return launch_head<2>(P, stream);
    case 3: return launch_head<3>(P, stream);
    default: return launch_head<4>(P, stream);
  }
}

extern "C" int dinvk_nchw_f32_to_nhwc_bf16(const float* in, void* out, int B, int C, int H, int W, int Cpad, float fill_scalar,
                                           const float* fill_batch, int has_fill, void* stream) {
  DINVK_CHECK_ARG(in && out && B >= 0 && C >= 1 && Cpad >= C + (has_fill ? 1 : 0) && Cpad % 8 == 0, "nchw_to_nhwc: bad arguments");
  if (B == 0) return DINVK_OK;
  const long long npix = (long long)B * H * W;
  const int grid = (int)std::min<long long>((npix + 255) / 256, (long long)sm_count() * 16);
  DINVK_LAUNCH(nchw_to_nhwc_kernel, dim3(grid), dim3(256), 0, stream, in, (bf16*)out, C, H, W, Cpad, fill_scalar, fill_batch, has_fill, npix);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_nhwc_bf16_to_nchw_f32(const void* in, const float* add, float* out, int B, int C, int H, int W, int Cpad,
                                           void* stream) {
  DINVK_CHECK_ARG(in && out && B >= 0 && C >= 1 && Cpad >= C, "nhwc_to_nchw: bad arguments");
  if (B == 0) return DINVK_OK;
  const long long npix = (long long)B * H * W;
  const int grid = (int)std::min<long long>((npix + 255) / 256, (long long)sm_count() * 16);
  DINVK_LAUNCH(nhwc_to_nchw_kernel, dim3(grid), dim3(256), 0, stream, (const bf16*)in, add, out, C, H, W, Cpad, npix);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_conv2x2_down_bf16(const void* x, const void* xadd, const void* weight, void* out, int B, int H, int W, int Cin,
                                       int Cout, void* stream) {
  DINVK_CHECK_ARG(x && weight && out && B >= 0 && H % 2 == 0 && W % 2 == 0, "conv2x2_down_bf16: bad arguments");
  if (B == 0) return DINVK_OK;
  if (!xadd && Cin % 64 == 0 && Cout % 64 == 0 && !getenv("DINVK_NO_TC_2X2"))
    return conv2x2_down_tc(x, weight, out, B, H, W, Cin, Cout, stream);
  const long long M = (long long)B * (H / 2) * (W / 2);
  DINVK_LAUNCH(conv2x2_bf16_kernel<false>, dim3((unsigned)ceil_div(M, 32), ceil_div(Cout, 64)), dim3(256), 0, stream, (const bf16*)x,
               (const bf16*)xadd, (const bf16*)weight, (bf16*)out, B, H, W, Cin, Cout);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_conv2x2_up_bf16(const void* x, const void* xadd, const void* weight, void* out, int B, int H, int W, int Cin,
                                     int Cout, void* stream) {
  DINVK_CHECK_ARG(x && weight && out && B >= 0, "conv2x2_up_bf16: bad arguments");
  if (B == 0) return DINVK_OK;
  if (!xadd && Cin % 64 == 0 && Cout % 64 == 0 && !getenv("DINVK_NO_TC_2X2"))
    return conv2x2_up_tc(x, weight, out, B, H, W, Cin, Cout, stream);
  const long long M = (long long)B * H * W;
  DINVK_LAUNCH(conv2x2_bf16_kernel<true>, dim3((unsigned)ceil_div(M, 32), ceil_div(4 * Cout, 64)), dim3(256), 0, stream, (const bf16*)x,
               (const bf16*)xadd, (const bf16*)weight, (bf16*)out, B, H, W, Cin, Cout);
  return DINVK_POST_LAUNCH();
}
