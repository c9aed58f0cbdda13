// conv_tc32.cu — fp32-grade tensor-core convolutions for the denoisers: split-operand wgmma implicit GEMM.
//
// The reference computes DRUNet / DnCNN in fp32 (deepinv/models/drunet.py:200-263, dncnn.py:121-140).  The bf16 path
// (conv_tc.cu) is fast but 3e-2 away from it; the CUDA-core path (conv_simt.cu) matches it but runs at a small fraction of
// the tensor peak.  Here every fp32 value v is carried as a pair (hi, lo) with hi + lo == v, and a product sum is evaluated
// as  sum a_hi*b_hi  +  sum (a_hi*b_lo + a_lo*b_hi)  on the tensor cores (fp32 accumulate): the dropped a_lo*b_lo term is
// 2^-22 relative.  The two sums live in separate accumulator columns ("main" and "corr"), and the accumulators are DRAINED
// into separate fp32 registers every `win` pipeline stages (round-to-nearest adds on the CUDA cores) so that the tensor
// core's accumulator rounding never sees more than a short partial sum.
//
// Activation layout in HBM ("split16"): NHWC with channels in blocks of 16, hi and lo interleaved per block:
//   x[b][y][x][c/16][p][c%16],  p = 0: hi, 1: lo      (fp32 words; 8 bytes per element; a pixel of a 16-channel block is
//   one 128-byte row = one swizzle row of the K-major wgmma operand).  hi + lo == v exactly, so residual / skip additions
//   read both words and lose nothing.
// Weight layout: per 64-row N tile 128 rows [W_hi (64 couts); W_lo (64 couts)], K-major, k = tap*Cin + c, both parts
//   rounded to tf32.
// One MMA "k step" on a 128-byte A row: steps 0,1 = the hi channels, steps 2,3 = the lo channels.
//   hi step: A_hi x [W_hi; W_lo]  (N = 128)  -> columns [0,64) main, [64,128) corr
//   lo step: A_lo x  W_hi         (N =  64)  -> columns [64,128) corr
// With wgmma's register accumulators the corr columns of the N = 128 fragment are exactly the registers of an N = 64
// fragment (registers 32..63), so the lo steps accumulate into the upper half of the same register array.
//
// Kernels (persistent, one CTA per SM): consumer warpgroups issue wgmma (M = 64 rows each), drain and run the epilogue
// from registers; one extra warp is the TMA producer.
#include "common.cuh"
#ifndef DINVK_EMUL
#include "tc_ptx.cuh"
#include <cuda_fp16.h>
#else
// host emulation (tests/emul): only the CUDA-core kernels of this file exist there — head, tail, layout converters; the 32-byte
// vector accesses of the store path are plain copies
namespace dinvk { namespace tc {
inline void ldg256(const void* p, uint32_t (&r)[8]) { std::memcpy(r, p, 32); }
inline void stg256(void* p, const uint32_t (&r)[8]) { std::memcpy(p, r, 32); }
} }
#endif

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace dinvk {
namespace t32 {

constexpr int TX = 16, TY = 8;             // pixel tile of one CTA: 16 x 8 = 128 GEMM rows
constexpr int A_TILE = 128 * 128;          // one 16-channel block of 128 pixels: 16 KB
constexpr int B_TILE = 128 * 128;          // [W_hi; W_lo] x 32 channels: 16 KB
constexpr int STAGE = 2 * A_TILE + B_TILE; // two channel blocks of one tap + their weights
constexpr int STAGES = 4;
constexpr int SMEM = STAGES * STAGE + 1024;
constexpr int THREADS = 2 * 128 + 32;      // two consumer warpgroups (GEMM rows [0, 64), [64, 128)) + the TMA producer warp

__device__ __forceinline__ float rna_tf32(float x) {
#ifndef DINVK_EMUL
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
#else
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);   // round to nearest, ties away: what cvt.rna does
#endif
}

// ---- the two split formats ------------------------------------------------------------------------------------------
// A 128-byte row block holds CH channels as [hi CH | lo CH].
//   FmtTF32 ("split16", fp32 words): hi = tf32(v) (cvt.rna), lo = v - hi (exact; the tensor core truncates it to tf32);
//            wgmma .tf32, K = 8 per MMA.  No range restriction.
//   FmtF16  ("split32h", fp16 words): hi = fp16(v), lo = fp16((v - hi) * 2^11) — the low part is scaled so that it sits in
//            fp16's normal range; the correction accumulators are weighted 2^-11 in the drain.  wgmma .f16, K = 16 per MMA: the
//            same 22-bit operands at TWICE the channels per MMA and half the bytes per element.  Range: |v| < 65504 — an
//            activation beyond it raises the sticky overflow flag and the network tail answers NaN (loud, never silent).
struct FmtTF32 {
  using elem = float;
  static constexpr int CH = 16, EB = 4, ID = 0;
  static constexpr float CORR = 1.0f;
#ifndef DINVK_EMUL
  static constexpr CUtensorMapDataType TM = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
#endif
};
struct FmtF16 {
  using elem = __half;
  static constexpr int CH = 32, EB = 2, ID = 1;
  static constexpr float CORR = 4.8828125e-4f;  // 2^-11
#ifndef DINVK_EMUL
  static constexpr CUtensorMapDataType TM = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
#endif
};

#ifndef DINVK_EMUL
template <class F, int N>
__device__ __forceinline__ void mma(float* d, uint32_t a_lo, uint32_t a_hi, uint32_t b_lo, uint32_t b_hi, uint32_t accumulate) {
  if constexpr (F::ID == 0) {
    if constexpr (N == 128) tc::wgmma_tf32_n128(d, a_lo, a_hi, b_lo, b_hi, accumulate);
    else tc::wgmma_tf32_n64(d, a_lo, a_hi, b_lo, b_hi, accumulate);
  } else {
    if constexpr (N == 128) tc::wgmma_f16_n128(d, a_lo, a_hi, b_lo, b_hi, accumulate);
    else tc::wgmma_f16_n64(d, a_lo, a_hi, b_lo, b_hi, accumulate);
  }
}
// one 128-byte A row block [hi CH | lo CH] (descriptor a) against the weight rows [W_hi; W_lo] at descriptor b (the block's
// CH channels): acc[0, 32) main += A_hi W_hi, acc[32, 64) corr += A_hi W_lo + A_lo W_hi.  `fresh` = 0 restarts both.
template <class F>
__device__ __forceinline__ void mma_block(float* acc, uint32_t a, uint32_t a_hi, uint32_t b, uint32_t b_hi, uint32_t fresh) {
  mma<F, 128>(acc, a, a_hi, b, b_hi, fresh);             // hi, first half of the block  x [W_hi; W_lo]
  mma<F, 128>(acc, a + 2, a_hi, b + 2, b_hi, 1u);        // hi, second half
  mma<F, 64>(acc + 32, a + 4, a_hi, b, b_hi, 1u);        // lo, first half  x W_hi
  mma<F, 64>(acc + 32, a + 6, a_hi, b + 2, b_hi, 1u);    // lo, second half
}
// v[i] (row 16 * (warp % 4) + lane / 4 + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + 2 * (lane % 4) + (i & 1)) += main + corr
template <class F>
__device__ __forceinline__ void drain(float* v, const float* acc) {
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] += acc[i] + acc[32 + i] * F::CORR;
}

// one warp's share of a consumed pipeline stage: the stage's `empty` barrier counts one arrival per consumer warp
__device__ __forceinline__ void release_stage(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) tc::mbar_arrive(bar);
}

struct Maps {
  CUtensorMap a[4];  // activation views: one (3x3, up) or one per tap (2x2 stride-2 down)
  CUtensorMap b;
};

struct Params {
  int B, H, W, Cin, Cout;   // H, W: the pixel grid the GEMM rows tile (3x3: image; down: OUTPUT grid; up: INPUT grid)
  int ntaps, kc_per_tap;    // kc_per_tap = Cin / (2 CH) (pipeline stages per tap)
  int dx[9], dy[9], amap[9];
  int mode;                 // 0: same-grid store; 2: 2x up-scatter (GEMM column = tap*Cout + co)
  int tiles_x, tiles_y, n_tiles;
  int relu;
  int win;                  // drain the accumulators every `win` stages
  const void* res;          // split layout, same shape as out
  const void* res2;
  void* out;                // split layout (B, Hout, Wout, Cout)
  int* flag;                // sticky overflow flag (FmtF16: an activation left the fp16 range), may be null
  const float* bias;
  int ngrp;                 // work-item order: `ngrp` N tiles (64 output channels each) of a pixel tile are ADJACENT work items, so that
                            // the CTAs that share its activations run at the same time and all but the first read them from L2
                            // (1 = all pixel tiles of N tile 0 first: every activation byte crosses HBM n_tiles times); divides n_tiles
};

// work item t -> (pixel tile, N tile): t = ((nt / g) * pixel_tiles + pt) * g + nt % g, g = P.ngrp
__device__ __forceinline__ void tile_index(const Params& P, int pixel_tiles, int t, int& pt, int& nt) {
  const int u = t / P.ngrp, lo = t - u * P.ngrp;
  const int hi = u / pixel_tiles;
  pt = u - hi * pixel_tiles;
  nt = hi * P.ngrp + lo;
}

#endif  // !DINVK_EMUL
// one channel block: v[CH] -> 128 bytes [hi CH | lo CH]; returns true if a value left the format's range
template <class F>
__device__ __forceinline__ bool store_split(typename F::elem* p, const float* v) {
  uint32_t u[4][8];
  bool bad = false;
  if constexpr (F::ID == 0) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float hi = rna_tf32(v[i]);
      u[i >> 3][i & 7] = __float_as_uint(hi);
      u[2 + (i >> 3)][i & 7] = __float_as_uint(v[i] - hi);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const __half h0 = __float2half_rn(v[i]), h1 = __float2half_rn(v[i + 1]);
      const __half l0 = __float2half_rn((v[i] - __half2float(h0)) * 2048.0f), l1 = __float2half_rn((v[i + 1] - __half2float(h1)) * 2048.0f);
      bad |= !(fabsf(v[i]) < 65000.0f) || !(fabsf(v[i + 1]) < 65000.0f);
      u[i >> 4][(i >> 1) & 7] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
      u[2 + (i >> 4)][(i >> 1) & 7] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
  }
  char* pc = reinterpret_cast<char*>(p);
#pragma unroll
  for (int k = 0; k < 4; ++k) tc::stg256(pc + 32 * k, u[k]);
  return bad;
}
// v[CH] += hi + lo of one block given as its four 32-byte chunks
template <class F>
__device__ __forceinline__ void add_split_raw(const uint32_t (*raw)[8], float* v) {
  if constexpr (F::ID == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] += __uint_as_float(raw[0][e]) + __uint_as_float(raw[2][e]);
      v[8 + e] += __uint_as_float(raw[1][e]) + __uint_as_float(raw[3][e]);
    }
  } else {
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&raw[c][e]));
        const float2 l = __half22float2(*reinterpret_cast<const __half2*>(&raw[2 + c][e]));
        v[c * 16 + 2 * e] += h.x + l.x * F::CORR;
        v[c * 16 + 2 * e + 1] += h.y + l.y * F::CORR;
      }
  }
}
template <class F>
__device__ __forceinline__ void add_split(const typename F::elem* p, float* v) {
  uint32_t raw[4][8];
  const char* pc = reinterpret_cast<const char*>(p);
#pragma unroll
  for (int k = 0; k < 4; ++k) tc::ldg256(pc + 32 * k, raw[k]);
  add_split_raw<F>(raw, v);
}

#ifndef DINVK_EMUL
// the same two conversions for one channel pair (c, c + 1), c even, as the wgmma epilogues hold them; p points at the hi
// element of channel c in its block (the lo element is CH further)
template <class F>
__device__ __forceinline__ void add_split_pair(const typename F::elem* p, float& a, float& b) {
  if constexpr (F::ID == 0) {
    const float2 h = __ldg(reinterpret_cast<const float2*>(p)), l = __ldg(reinterpret_cast<const float2*>(p + F::CH));
    a += h.x + l.x;
    b += h.y + l.y;
  } else {
    const float2 h = __half22float2(__ldg(reinterpret_cast<const __half2*>(p)));
    const float2 l = __half22float2(__ldg(reinterpret_cast<const __half2*>(p + F::CH)));
    a += h.x + l.x * F::CORR;
    b += h.y + l.y * F::CORR;
  }
}
template <class F>
__device__ __forceinline__ bool store_split_pair(typename F::elem* p, float a, float b) {
  if constexpr (F::ID == 0) {
    const float ha = rna_tf32(a), hb = rna_tf32(b);
    *reinterpret_cast<float2*>(p) = make_float2(ha, hb);
    *reinterpret_cast<float2*>(p + F::CH) = make_float2(a - ha, b - hb);
    return false;
  } else {
    const __half h0 = __float2half_rn(a), h1 = __float2half_rn(b);
    const __half l0 = __float2half_rn((a - __half2float(h0)) * 2048.0f), l1 = __float2half_rn((b - __half2float(h1)) * 2048.0f);
    *reinterpret_cast<__half2*>(p) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(p + F::CH) = __halves2half2(l0, l1);
    return !(fabsf(a) < 65000.0f) || !(fabsf(b) < 65000.0f);
  }
}

// epilogue of the drained sums v (see drain) of one m64 x 64-column block: bias, ReLU, residuals, split store.  The caller
// maps the thread's two rows to pixels; n0 = first GEMM column of the N tile.
template <class F>
__device__ __forceinline__ void epilogue_split(const Params& P, float* v, int b, const int (&y)[2], const int (&x)[2], int n0) {
  using E = typename F::elem;
  const int q = threadIdx.x & 3;
  const int tap = P.mode == 2 ? n0 / P.Cout : 0;
  const int c0 = n0 - tap * P.Cout;   // output channel of GEMM column n0
  bool bad = false;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!(y[r] < P.H && x[r] < P.W)) continue;
    long long pix;   // output pixel index
    if (P.mode == 2) pix = ((long long)b * (2 * P.H) + 2 * y[r] + (tap >> 1)) * (2LL * P.W) + 2 * x[r] + (tap & 1);
    else pix = ((long long)b * P.H + y[r]) * P.W + x[r];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + 8 * j + 2 * q;
      float a = v[4 * j + 2 * r], bb = v[4 * j + 2 * r + 1];
      if (P.bias) { a += __ldg(P.bias + c); bb += __ldg(P.bias + c + 1); }
      if (P.relu) { a = fmaxf(a, 0.f); bb = fmaxf(bb, 0.f); }
      const long long o = pix * P.Cout * 2 + (c / F::CH) * 2 * F::CH + (c % F::CH);
      if (P.res) add_split_pair<F>(static_cast<const E*>(P.res) + o, a, bb);
      if (P.res2) add_split_pair<F>(static_cast<const E*>(P.res2) + o, a, bb);
      bad |= store_split_pair<F>(static_cast<E*>(P.out) + o, a, bb);
    }
  }
  if (bad && P.flag) atomicOr(P.flag, 1);
}

template <class F>
__global__ void __launch_bounds__(THREADS, 1) conv_tc32_kernel(const __grid_constant__ Maps M, const Params P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pixel_tiles = P.B * P.tiles_y * P.tiles_x;
  const int total_tiles = pixel_tiles * P.n_tiles;
  const int nk = P.ntaps * P.kc_per_tap;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&M.a[0]);
    tc::prefetch_tmap(&M.b);
    for (int s = 0; s < STAGES; ++s) { tc::mbar_init(&full_bar[s], 1); tc::mbar_init(&empty_bar[s], 8); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int pt, nt; tile_index(P, pixel_tiles, t, pt, nt);
        const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
        const int y0 = (r / P.tiles_x) * TY, x0 = (r % P.tiles_x) * TX;
        for (int kb = 0; kb < nk; ++kb) {
          const int tap = kb / P.kc_per_tap, kc = kb - tap * P.kc_per_tap;
          tc::mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * STAGE;
          tc::mbar_arrive_expect_tx(&full_bar[s], STAGE);
          // channel blocks 2kc and 2kc+1: one 128-byte row ([hi CH | lo CH]) each, at element offset 2 CH * block
          tc::tma_load_4d(sa, &M.a[P.amap[tap]], &full_bar[s], (2 * kc) * (2 * F::CH), x0 + P.dx[tap], y0 + P.dy[tap], b);
          tc::tma_load_4d(sa + A_TILE, &M.a[P.amap[tap]], &full_bar[s], (2 * kc + 1) * (2 * F::CH), x0 + P.dx[tap], y0 + P.dy[tap], b);
          tc::tma_load_2d(sa + 2 * A_TILE, &M.b, &full_bar[s], tap * P.Cin + kc * (2 * F::CH), nt * 128);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: wgmma, drains, epilogue =====================
    const int wg = warp >> 2;
    constexpr uint32_t HI = tc::desc_hi_sw128(1024);
    const uint32_t smem_lo = tc::smem_u32(smem) >> 4;
    float acc[64], v[32];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int pt, nt; tile_index(P, pixel_tiles, t, pt, nt);
      const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
      const int y0 = (r / P.tiles_x) * TY, x0 = (r % P.tiles_x) * TX;
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = 0.f;
      int in_win = 0, pend = -1;
      for (int kb = 0; kb < nk; ++kb) {
        tc::mbar_wait(&full_bar[s], ph);
        const uint32_t a0 = smem_lo + static_cast<uint32_t>(s) * (STAGE >> 4) + static_cast<uint32_t>(wg * (64 * 128 >> 4));
        const uint32_t b0 = smem_lo + static_cast<uint32_t>(s) * (STAGE >> 4) + (2 * A_TILE >> 4);
        tc::wgmma_fence();
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)  // B: second channel block = +64 bytes inside the weight row
          mma_block<F>(acc, a0 + jj * (A_TILE >> 4), HI, b0 + jj * 4, HI, (jj | in_win) != 0 ? 1u : 0u);
        tc::wgmma_commit();
        if (++in_win == P.win || kb == nk - 1) {
          tc::wgmma_wait<0>();
          tc::reg_fence<64>(acc);
          if (pend >= 0) release_stage(&empty_bar[pend]);
          release_stage(&empty_bar[s]);
          pend = -1;
          drain<F>(v, acc);
          in_win = 0;
        } else {
          tc::wgmma_wait<1>();
          if (pend >= 0) release_stage(&empty_bar[pend]);
          pend = s;
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      int y[2], x[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * rr;
        y[rr] = y0 + m / TX; x[rr] = x0 + m % TX;
      }
      epilogue_split<F>(P, v, b, y, x, nt * 64);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 3x3 convolution with HALO REUSE (the body layers: almost all of a DRUNet forward).
//
// The per-tap kernel above re-reads every activation tile 9 times and every weight tile once per 128 pixels.  Here a CTA
// owns an (8 MH) x 16-pixel tile.  Per 16-channel block ONE TMA box brings the (8 MH + 8) x (16 + 2)-position slab (tile +
// halo; out-of-range positions zero-filled = the convolution's padding; a multiple of 8 positions per slab row keeps every
// 8-position group 1024-byte periodic) of [hi | lo] rows into shared memory, and the nine taps are nine shifted wgmma
// descriptors into it (start + (ky * SLAB_X + kx) * 128 B, stride between 8-row groups = one slab row); the 128-byte swizzle
// is a function of the shared-memory address bits, so the shifted starts need no base offset.  A weight tile holds TWO taps
// of one channel block ([tap even | tap odd] per row, rows = [W_hi; W_lo]) and is shared by all consumer warpgroups.
// Consumer warpgroup g owns the m64 block (x-half g / 2, y-half g % 2) = 8 x 8 pixels; a window = `win` channel blocks.
// ---------------------------------------------------------------------------------------------------------------
namespace slab {
constexpr int TYP = 16;                           // CTA pixel tile height
constexpr int SLAB_Y = TYP + 2;
constexpr int A_STAGES = 2, B_STAGES = 6;
constexpr int WT_TILE = 128 * 128;
template <int MH> struct Geom {
  static constexpr int TXP = 8 * MH;              // CTA pixel tile width
  static constexpr int SLAB_X = TXP + 8;
  static constexpr int SLAB_BYTES = SLAB_X * SLAB_Y * 128;
  static constexpr int SMEM_BYTES = A_STAGES * SLAB_BYTES + B_STAGES * WT_TILE + 1024;
  static constexpr int NWG = 2 * MH;
  static constexpr int THREADS = 128 * NWG + 32;
  static_assert(SLAB_BYTES % 1024 == 0, "slab stages must stay 1024-byte aligned");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};
}  // namespace slab

template <class F, int MH>
__global__ void __launch_bounds__(slab::Geom<MH>::THREADS, 1) conv_tc32_slab_kernel(const __grid_constant__ Maps M, const Params P) {
  using namespace slab;
  using G = Geom<MH>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_b = smem + A_STAGES * G::SLAB_BYTES;
  __shared__ __align__(8) uint64_t afull[A_STAGES];
  __shared__ __align__(8) uint64_t aempty[A_STAGES];
  __shared__ __align__(8) uint64_t bfull[B_STAGES];
  __shared__ __align__(8) uint64_t bempty[B_STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pixel_tiles = P.B * P.tiles_y * P.tiles_x;
  const int total_tiles = pixel_tiles * P.n_tiles;
  const int nblk = P.Cin / F::CH;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&M.a[0]);
    tc::prefetch_tmap(&M.b);
    for (int s = 0; s < A_STAGES; ++s) { tc::mbar_init(&afull[s], 1); tc::mbar_init(&aempty[s], 4 * G::NWG); }
    for (int s = 0; s < B_STAGES; ++s) { tc::mbar_init(&bfull[s], 1); tc::mbar_init(&bempty[s], 4 * G::NWG); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 * G::NWG) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int sa = 0; uint32_t pha = 0;
      int sb = 0; uint32_t phb = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int pt, nt; tile_index(P, pixel_tiles, t, pt, nt);
        const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
        const int y0 = (r / P.tiles_x) * TYP, x0 = (r % P.tiles_x) * G::TXP;
        for (int j = 0; j < nblk; ++j) {
          tc::mbar_wait(&aempty[sa], pha ^ 1);
          tc::mbar_arrive_expect_tx(&afull[sa], G::SLAB_BYTES);
          tc::tma_load_4d(smem + sa * G::SLAB_BYTES, &M.a[0], &afull[sa], j * (2 * F::CH), x0 - 1, y0 - 1, b);
          if (++sa == A_STAGES) { sa = 0; pha ^= 1; }
          for (int tp = 0; tp < 5; ++tp) {
            tc::mbar_wait(&bempty[sb], phb ^ 1);
            tc::mbar_arrive_expect_tx(&bfull[sb], WT_TILE);
            tc::tma_load_2d(smem_b + sb * WT_TILE, &M.b, &bfull[sb], (j * 5 + tp) * (2 * F::CH), nt * 128);
            if (++sb == B_STAGES) { sb = 0; phb ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers =====================
    // The tap loop is fully unrolled (compile-time tap shifts, one barrier wait and one commit per weight tile).  The group of
    // weight tile i is committed before the group of tile i - 1 is waited for; stages are released once their group completed.
    const int wg = warp >> 2;
    const int half = wg >> 1, yh = wg & 1;
    constexpr uint32_t HI_A = tc::desc_hi_sw128(G::SLAB_X * 128);
    constexpr uint32_t HI_B = tc::desc_hi_sw128(1024);
    const uint32_t slab_lo0 = (tc::smem_u32(smem) >> 4) + static_cast<uint32_t>((8 * yh * G::SLAB_X + 8 * half) * 8);
    const uint32_t bt_lo0 = tc::smem_u32(smem_b) >> 4;
    float acc[64], v[32];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int sa = 0; uint32_t pha = 0;
    int sb = 0; uint32_t phb = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int pt, nt; tile_index(P, pixel_tiles, t, pt, nt);
      const int b = pt / (P.tiles_y * P.tiles_x), r = pt - b * (P.tiles_y * P.tiles_x);
      const int y0 = (r / P.tiles_x) * TYP, x0 = (r % P.tiles_x) * G::TXP;
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = 0.f;
      int in_win = 0;  // channel blocks accumulated in the current window
      int pend_a = -1, pend_b = -1;
      for (int j = 0; j < nblk; ++j) {
        tc::mbar_wait(&afull[sa], pha);
        const uint32_t slab_lo = slab_lo0 + static_cast<uint32_t>(sa) * (G::SLAB_BYTES >> 4);
        const uint32_t fresh = in_win == 0 ? 0u : 1u;
        const bool last_of_win = (in_win + 1 == P.win) || (j == nblk - 1);
#pragma unroll
        for (int tp = 0; tp < 5; ++tp) {
          tc::mbar_wait(&bfull[sb], phb);
          const uint32_t b_lo = bt_lo0 + static_cast<uint32_t>(sb) * (WT_TILE >> 4);
          tc::wgmma_fence();
#pragma unroll
          for (int par = 0; par < 2; ++par) {
            const int tap = 2 * tp + par;
            if (tap < 9) {
              const uint32_t a_t = slab_lo + static_cast<uint32_t>(((tap / 3) * G::SLAB_X + (tap % 3)) * 8);
              mma_block<F>(acc, a_t, HI_A, b_lo + par * 4, HI_B, tap == 0 ? fresh : 1u);  // odd tap: +64 bytes inside the weight row
            }
          }
          tc::wgmma_commit();
          if (tp == 4 && last_of_win) {
            tc::wgmma_wait<0>();
            tc::reg_fence<64>(acc);
            if (pend_b >= 0) release_stage(&bempty[pend_b]);
            if (pend_a >= 0) release_stage(&aempty[pend_a]);
            release_stage(&bempty[sb]);
            release_stage(&aempty[sa]);
            pend_a = -1; pend_b = -1;
            drain<F>(v, acc);
          } else {
            tc::wgmma_wait<1>();
            if (pend_b >= 0) release_stage(&bempty[pend_b]);
            if (pend_a >= 0) release_stage(&aempty[pend_a]);
            pend_b = sb;
            pend_a = tp == 4 ? sa : -1;
          }
          if (++sb == B_STAGES) { sb = 0; phb ^= 1; }
        }
        if (++sa == A_STAGES) { sa = 0; pha ^= 1; }
        in_win = last_of_win ? 0 : in_win + 1;
      }
      int y[2], x[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = 16 * (warp & 3) + (lane >> 2) + 8 * rr;
        y[rr] = y0 + 8 * yh + (m >> 3); x[rr] = x0 + 8 * half + (m & 7);
      }
      epilogue_split<F>(P, v, b, y, x, nt * 64);
    }
  }
}

#endif  // !DINVK_EMUL
// ---------------------------------------------------------------------------------------------------------------
// Network HEAD (CUDA cores; 0.1 % of the FLOPs, bound by its 8-byte-per-element output write): 3x3 convolution from the
// reference's NCHW fp32 image (+ optional constant noise-level channel, drunet.py:190-200) to Cout split16 channels.
// One thread per pixel: its 9*CT inputs sit in registers, the weights in shared memory (every lane reads the same
// word: broadcast).
// ---------------------------------------------------------------------------------------------------------------
struct HeadParams {
  const float* x; const float* w; const float* bias; void* out;
  int B, C, H, W, Cout;
  float fill_scalar; const float* fill_batch; int has_fill; int relu;
  int* flag;
};

template <class F, int CT>
__global__ void __launch_bounds__(256) head_tc32_kernel(const HeadParams P) {
  // weights [Cout][KP] in shared memory, KP = 9*CT rounded up to a multiple of 4: one 128-bit broadcast load feeds four FMAs
  // (the first version read one word per FMA and was bound by the shared-memory pipe: 1.0 ms instead of the 0.3 ms its writes take)
  constexpr int KR = 9 * CT, KP = (KR + 3) & ~3;
#ifndef DINVK_EMUL
  extern __shared__ __align__(16) float sw[];  // module layout (Cout, CT, 3, 3) -> sw[co * KP + c * 9 + tap], zero padded
#else
  float* sw = reinterpret_cast<float*>(::emul::dyn_smem());
#endif
  for (int i = threadIdx.x; i < P.Cout * KP; i += blockDim.x) {
    const int co = i / KP, k = i - co * KP;
    sw[i] = k < KR ? __ldg(P.w + co * KR + k) : 0.f;
  }
  __syncthreads();
  const long long npix = (long long)P.B * P.H * P.W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const long long HW = (long long)P.H * P.W;
  const int b = (int)(p / HW);
  const int rem = (int)(p - (long long)b * HW);
  const int y = rem / P.W, x = rem - y * P.W;
  const float fillv = P.has_fill ? (P.fill_batch ? __ldg(P.fill_batch + b) : P.fill_scalar) : 0.f;
  float in[KP];
#pragma unroll
  for (int k = KR; k < KP; ++k) in[k] = 0.f;
  const float* img = P.x + (long long)b * P.C * HW;
#pragma unroll
  for (int c = 0; c < CT; ++c) {
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
      const bool inb = (yy >= 0) && (yy < P.H) && (xx >= 0) && (xx < P.W);
      float val = 0.f;
      if (inb) val = (c < P.C) ? __ldg(img + (long long)c * HW + (long long)yy * P.W + xx) : fillv;
      in[c * 9 + tap] = val;
    }
  }
  typename F::elem* o = static_cast<typename F::elem*>(P.out) + p * P.Cout * 2;
  bool bad = false;
  for (int c0 = 0; c0 < P.Cout; c0 += F::CH) {
    float v[F::CH];
#pragma unroll
    for (int i = 0; i < F::CH; ++i) {
      float a = P.bias ? __ldg(P.bias + c0 + i) : 0.f;
      const float4* wr = reinterpret_cast<const float4*>(sw + (c0 + i) * KP);
#pragma unroll
      for (int k = 0; k < KP / 4; ++k) {
        const float4 w4 = wr[k];
        a = fmaf(in[4 * k], w4.x, a); a = fmaf(in[4 * k + 1], w4.y, a);
        a = fmaf(in[4 * k + 2], w4.z, a); a = fmaf(in[4 * k + 3], w4.w, a);
      }
      v[i] = P.relu ? fmaxf(a, 0.f) : a;
    }
    bad |= store_split<F>(o + c0 * 2, v);
  }
  if (bad && P.flag) atomicOr(P.flag, 1);
}

// HEAD for Cout = 64: lanes = output channels.  A warp owns 32 consecutive pixels of two image rows; lane l computes
// channels (2l, 2l+1) of every pixel with its 2 * 9 * CT weights in registers.  The 3 x 3 x CT inputs of the 32 pixels
// are loaded once (lane i holds column x0 + i of the three rows; lanes 0 / 1 also hold the two halo columns) and
// broadcast by shuffles while the warp slides along the row.  A pixel's 64 channels leave as four coalesced
// 64-byte (fp16) / 128-byte (tf32) segments: [hi | lo] of each channel block.  (The thread-per-pixel version above
// stores 128 bytes per lane at a 256-byte stride and reads its weights through the shared-memory pipe: 0.9 ms.)
template <class F, int CT>
__global__ void __launch_bounds__(256) head64_tc32_kernel(const HeadParams P) {
  using E = typename F::elem;
  constexpr int R = 2;   // output rows per warp: rows y0, y0 + 1 share two of their three input rows (6 instead of 9 shuffles per pixel)
  const int lane = threadIdx.x & 31;
  const int segs = (P.W + 31) / 32, rows2 = (P.H + R - 1) / R;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)P.B * rows2 * segs) return;
  const int b = (int)(wid / ((long long)rows2 * segs)), rem = (int)(wid - (long long)b * rows2 * segs);
  const int y0 = (rem / segs) * R, x0 = (rem % segs) * 32;
  float w0[CT * 9], w1[CT * 9];
#pragma unroll
  for (int k = 0; k < CT * 9; ++k) {
    w0[k] = __ldg(P.w + (long long)(2 * lane) * CT * 9 + k);
    w1[k] = __ldg(P.w + (long long)(2 * lane + 1) * CT * 9 + k);
  }
  const float b0 = P.bias ? __ldg(P.bias + 2 * lane) : 0.f, b1 = P.bias ? __ldg(P.bias + 2 * lane + 1) : 0.f;
  const float fillv = P.has_fill ? (P.fill_batch ? __ldg(P.fill_batch + b) : P.fill_scalar) : 0.f;
  const long long HW = (long long)P.H * P.W;
  const float* img = P.x + (long long)b * P.C * HW;
  // mid[c][r]: column x0 + lane of input row y0 - 1 + r; edge[c][r]: lane 0 holds column x0 - 1, lane 1 column x0 + 32
  float mid[CT][R + 2], edge[CT][R + 2];
  const int xe = lane == 0 ? x0 - 1 : x0 + 32;
#pragma unroll
  for (int c = 0; c < CT; ++c)
#pragma unroll
    for (int r = 0; r < R + 2; ++r) {
      const int yy = y0 + r - 1;
      const bool rowin = yy >= 0 && yy < P.H;
      const int xm = x0 + lane;
      float m = 0.f, e = 0.f;
      if (rowin && xm < P.W) m = c < P.C ? __ldg(img + (long long)c * HW + (long long)yy * P.W + xm) : fillv;
      if (rowin && lane < 2 && xe >= 0 && xe < P.W) e = c < P.C ? __ldg(img + (long long)c * HW + (long long)yy * P.W + xe) : fillv;
      mid[c][r] = m; edge[c][r] = e;
    }
  const int eo = ((2 * lane) / F::CH) * 2 * F::CH + (2 * lane) % F::CH;
  E* orow = static_cast<E*>(P.out) + (((long long)b * P.H + y0) * P.W + x0) * 128 + eo;
  const long long rstride = (long long)P.W * 128;
  bool bad = false;
  // sliding window of the three columns around pixel p
  float cl[CT][R + 2], cc[CT][R + 2], cr[CT][R + 2], last[CT][R + 2];
#pragma unroll
  for (int c = 0; c < CT; ++c)
#pragma unroll
    for (int r = 0; r < R + 2; ++r) {
      cl[c][r] = __shfl_sync(0xffffffffu, edge[c][r], 0);
      cc[c][r] = __shfl_sync(0xffffffffu, mid[c][r], 0);
      last[c][r] = __shfl_sync(0xffffffffu, edge[c][r], 1);
    }
  const int npx = min(32, P.W - x0);
#pragma unroll 1
  for (int p = 0; p < npx; ++p) {
#pragma unroll
    for (int c = 0; c < CT; ++c)
#pragma unroll
      for (int r = 0; r < R + 2; ++r) {
        const float nm = __shfl_sync(0xffffffffu, mid[c][r], (p + 1) & 31);
        cr[c][r] = p == 31 ? last[c][r] : nm;
      }
#pragma unroll
    for (int ro = 0; ro < R; ++ro) {
      float a0 = b0, a1 = b1;
#pragma unroll
      for (int c = 0; c < CT; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          a0 = fmaf(w0[c * 9 + ky * 3 + 0], cl[c][ro + ky], a0); a1 = fmaf(w1[c * 9 + ky * 3 + 0], cl[c][ro + ky], a1);
          a0 = fmaf(w0[c * 9 + ky * 3 + 1], cc[c][ro + ky], a0); a1 = fmaf(w1[c * 9 + ky * 3 + 1], cc[c][ro + ky], a1);
          a0 = fmaf(w0[c * 9 + ky * 3 + 2], cr[c][ro + ky], a0); a1 = fmaf(w1[c * 9 + ky * 3 + 2], cr[c][ro + ky], a1);
        }
      if (P.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
      if (y0 + ro < P.H) {
        E* o = orow + ro * rstride + (long long)p * 128;
        if constexpr (F::ID == 0) {
          const float h0 = rna_tf32(a0), h1 = rna_tf32(a1);
          *reinterpret_cast<float2*>(o) = make_float2(h0, h1);
          *reinterpret_cast<float2*>(o + F::CH) = make_float2(a0 - h0, a1 - h1);
        } else {
          const __half2 h = __floats2half2_rn(a0, a1);
          const float2 hf = __half22float2(h);
          const __half2 l = __floats2half2_rn((a0 - hf.x) * 2048.0f, (a1 - hf.y) * 2048.0f);
          bad |= !(fmaxf(fabsf(a0), fabsf(a1)) < 65000.0f);
          *reinterpret_cast<__half2*>(o) = h;
          *reinterpret_cast<__half2*>(o + F::CH) = l;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CT; ++c)
#pragma unroll
      for (int r = 0; r < R + 2; ++r) { cl[c][r] = cc[c][r]; cc[c][r] = cr[c][r]; }
  }
  if (bad && P.flag) atomicOr(P.flag, 1);
}

// ---------------------------------------------------------------------------------------------------------------
// Network TAIL (CUDA cores): 3x3 convolution from C split16 channels to Cout <= 4 channels, fp32 NCHW output
// (+ bias, + optional NCHW term: DnCNN's "+ x", dncnn.py:138).  A CTA stages the (32+2) x (8+2) halo tile as
// v = hi + lo in shared memory ([position][C + 4] words: 128-bit loads by adjacent pixels are conflict-free).
// ---------------------------------------------------------------------------------------------------------------
struct TailParams {
  const void* x; const float* w; const float* bias; const float* add; float* out;
  int B, H, W, C, Cout;
  const int* flag;   // overflow flag of the network (FmtF16): set -> the output is NaN
};
constexpr int TL_TX = 32, TL_TY = 8;

template <class F, int CO>
__global__ void __launch_bounds__(256) tail_tc32_kernel(const TailParams P) {
#ifndef DINVK_EMUL
  extern __shared__ __align__(16) float sm[];
#else
  float* sm = reinterpret_cast<float*>(::emul::dyn_smem());
#endif
  const int C = P.C, CP = C + 4;
  float* sx = sm;                                   // (TL_TY+2)*(TL_TX+2) positions x CP
  float* swt = sm + (TL_TY + 2) * (TL_TX + 2) * CP;  // [co][tap][C]
  const int tiles_x = (P.W + TL_TX - 1) / TL_TX, tiles_y = (P.H + TL_TY - 1) / TL_TY;
  const int b = blockIdx.x / (tiles_x * tiles_y), r = blockIdx.x - b * (tiles_x * tiles_y);
  const int y0 = (r / tiles_x) * TL_TY, x0 = (r % tiles_x) * TL_TX;
  // weights (Cout, C, 3, 3) -> [co][tap][c]
  for (int i = threadIdx.x; i < CO * 9 * C; i += blockDim.x) {
    const int co = i / (9 * C), rem = i - co * 9 * C, tap = rem / C, c = rem - tap * C;
    swt[i] = __ldg(P.w + ((long long)co * C + c) * 9 + tap);
  }
  // halo tile: one float4 of hi + one of lo per (position, 4 channels)
  const int npos = (TL_TY + 2) * (TL_TX + 2), q4 = C / 4;
  for (int i = threadIdx.x; i < npos * q4; i += blockDim.x) {
    const int pos = i / q4, cq = i - pos * q4;
    const int yy = y0 + pos / (TL_TX + 2) - 1, xx = x0 + pos % (TL_TX + 2) - 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (yy >= 0 && yy < P.H && xx >= 0 && xx < P.W) {
      const int c = cq * 4, blk = c / F::CH, ib = c % F::CH;
      const typename F::elem* src = static_cast<const typename F::elem*>(P.x) + (((long long)b * P.H + yy) * P.W + xx) * C * 2 + blk * 2 * F::CH + ib;
      if constexpr (F::ID == 0) {
        const float4 h = __ldg(reinterpret_cast<const float4*>(src));
        const float4 l = __ldg(reinterpret_cast<const float4*>(src + F::CH));
        v = make_float4(h.x + l.x, h.y + l.y, h.z + l.z, h.w + l.w);
      } else {
        const uint2 hu = __ldg(reinterpret_cast<const uint2*>(src)), lu = __ldg(reinterpret_cast<const uint2*>(src + F::CH));
        const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&hu.x)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&hu.y));
        const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&lu.x)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&lu.y));
        v = make_float4(h0.x + l0.x * F::CORR, h0.y + l0.y * F::CORR, h1.x + l1.x * F::CORR, h1.y + l1.y * F::CORR);
      }
    }
    *reinterpret_cast<float4*>(sx + pos * CP + cq * 4) = v;
  }
  __syncthreads();
  const int ty = threadIdx.x / TL_TX, tx = threadIdx.x % TL_TX;
  const int y = y0 + ty, x = x0 + tx;
  float acc[CO];
#pragma unroll
  for (int co = 0; co < CO; ++co) acc[co] = 0.f;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const float* px = sx + ((ty + tap / 3) * (TL_TX + 2) + tx + tap % 3) * CP;
#pragma unroll 4
    for (int c = 0; c < C; c += 4) {
      const float4 a = *reinterpret_cast<const float4*>(px + c);
#pragma unroll
      for (int co = 0; co < CO; ++co) {
        const float4 w4 = *reinterpret_cast<const float4*>(swt + (co * 9 + tap) * C + c);
        acc[co] = fmaf(a.x, w4.x, acc[co]); acc[co] = fmaf(a.y, w4.y, acc[co]);
        acc[co] = fmaf(a.z, w4.z, acc[co]); acc[co] = fmaf(a.w, w4.w, acc[co]);
      }
    }
  }
  const bool poisoned = P.flag && *reinterpret_cast<const volatile int*>(P.flag) != 0;
  if (y < P.H && x < P.W) {
#pragma unroll
    for (int co = 0; co < CO; ++co) {
      if (co < P.Cout) {
        const long long o = (((long long)b * P.Cout + co) * P.H + y) * P.W + x;
        float val = acc[co] + (P.bias ? __ldg(P.bias + co) : 0.f);
        if (P.add) val += __ldg(P.add + o);
        if (poisoned) val = __uint_as_float(0x7fc00000u);   // an activation left the fp16 range somewhere in this network: NaN
        P.out[o] = val;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// TAIL for C = 64 (every DRUNet / DnCNN of the reference): lanes = channels.  A warp owns a strip of WT = 16 / CO output
// columns and walks TL_RC output rows downwards; lane l carries channels (2l, 2l+1): its 2 * 9 * CO weights stay in
// registers for the whole kernel, an input pixel is ONE coalesced 256-byte (fp16) / 512-byte (tf32) row per warp, read
// once per strip (no shared memory, no staging phase), and contributes to the 3 x 3 outputs around it.  The per-lane
// partial sums of an output row (WT * CO = 16 values) are summed across the 32 lanes by a transposing butterfly
// (8 + 4 + 2 + 1 + 1 shuffles: each step halves the values a lane keeps), after which lane 2v owns value v.
// The first version (thread = pixel, halo tile and weights in shared memory: tail_tc32_kernel) spent 3 LDS.128 per
// 8 FMAs and took 1.4 ms for 64 x 256^2; this one is bound by its 1152 FMAs per pixel.
// ---------------------------------------------------------------------------------------------------------------
constexpr int TL_RC = 32;  // output rows per warp

template <int N>
__device__ __forceinline__ void halve_across(float (&a)[16], int upper, int offset) {
#pragma unroll
  for (int j = 0; j < N / 2; ++j) {
    const float send = upper ? a[j] : a[j + N / 2];
    const float keep = upper ? a[j + N / 2] : a[j];
    a[j] = keep + __shfl_xor_sync(0xffffffffu, send, offset);
  }
}

// input row r of the strip: the lane's two channels (raw hi / lo words) of the WT + 2 columns xs - 1 .. xs + WT.  The loads are
// UNCONDITIONAL (clamped addresses; out-of-image values are zeroed when they are converted) and fill plain register arrays, so
// that all 2 (WT + 2) of them are in flight together — the first version converted each pixel right after its two loads and
// ran one memory round trip per pixel: 2.0 ms instead of the 1.1 ms of the version before it.
template <class F> struct TailRaw { using type = uint32_t; };
template <> struct TailRaw<FmtTF32> { using type = float2; };

template <class F, int WT>
__device__ __forceinline__ void tail_load_raw(const typename F::elem* img, int r, int xs, int H, int W, typename TailRaw<F>::type (&rh)[WT + 2],
                                              typename TailRaw<F>::type (&rl)[WT + 2]) {
  using R = typename TailRaw<F>::type;
  const int rc = min(max(r, 0), H - 1);
#pragma unroll
  for (int i = 0; i < WT + 2; ++i) {
    const int xc = min(max(xs - 1 + i, 0), W - 1);
    const typename F::elem* q = img + ((long long)rc * W + xc) * 128;
    rh[i] = __ldg(reinterpret_cast<const R*>(q));
    rl[i] = __ldg(reinterpret_cast<const R*>(q + F::CH));
  }
}
template <class F, int WT>
__device__ __forceinline__ void tail_convert(bool rowin, int xs, int W, const typename TailRaw<F>::type (&rh)[WT + 2],
                                             const typename TailRaw<F>::type (&rl)[WT + 2], float (&v0)[WT + 2], float (&v1)[WT + 2]) {
#pragma unroll
  for (int i = 0; i < WT + 2; ++i) {
    const int x = xs - 1 + i;
    const bool in = rowin && x >= 0 && x < W;
    float a, b;
    if constexpr (F::ID == 0) {
      a = rh[i].x + rl[i].x; b = rh[i].y + rl[i].y;
    } else {
      const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&rh[i])), l = __half22float2(*reinterpret_cast<const __half2*>(&rl[i]));
      a = fmaf(l.x, F::CORR, h.x); b = fmaf(l.y, F::CORR, h.y);
    }
    v0[i] = in ? a : 0.f; v1[i] = in ? b : 0.f;
  }
}
// input row t (image row r0 - 1 + t) feeds output rows t + 1, t, t - 1 (ky = 0, 1, 2); PH = t % 3 names the accumulator slots;
// afterwards output row t - 1 is complete: summed over the lanes, written, its slot cleared
template <int CO, int PH>
__device__ __forceinline__ void tail_row(const TailParams& P, int t, int tmax, int b, int r0, int xs, int lane, bool poisoned,
                                         const float (&w0)[CO][9], const float (&w1)[CO][9], float (&acc)[3][16],
                                         const float (&v0)[16 / CO + 2], const float (&v1)[16 / CO + 2]) {
  constexpr int WT = 16 / CO;
  if (t > tmax) return;
  const int r = r0 - 1 + t;
  if (r >= 0 && r < P.H) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      constexpr int S0 = (PH + 1) % 3, S1 = PH, S2 = (PH + 2) % 3;
      float* a = ky == 0 ? acc[S0] : (ky == 1 ? acc[S1] : acc[S2]);
#pragma unroll
      for (int co = 0; co < CO; ++co)
#pragma unroll
        for (int j = 0; j < WT; ++j) {
          float s = a[co * WT + j];
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            s = fmaf(w0[co][ky * 3 + kx], v0[j + kx], s);
            s = fmaf(w1[co][ky * 3 + kx], v1[j + kx], s);
          }
          a[co * WT + j] = s;
        }
    }
  }
  constexpr int SD = (PH + 2) % 3;
  const int y = r0 + t - 2;
  if (t >= 2 && y < P.H) {
    float red[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) red[i] = acc[SD][i];
    halve_across<16>(red, lane & 16, 16);
    halve_across<8>(red, lane & 8, 8);
    halve_across<4>(red, lane & 4, 4);
    halve_across<2>(red, lane & 2, 2);
    const float tot = red[0] + __shfl_xor_sync(0xffffffffu, red[0], 1);
    const int vi = lane >> 1, co = vi / WT, x = xs + vi % WT;
    if (!(lane & 1) && co < P.Cout && x < P.W) {
      const long long o = (((long long)b * P.Cout + co) * P.H + y) * P.W + x;
      float val = tot + (P.bias ? __ldg(P.bias + co) : 0.f);
      if (P.add) val += __ldg(P.add + o);
      if (poisoned) val = __uint_as_float(0x7fc00000u);
      P.out[o] = val;
    }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[SD][i] = 0.f;
}

template <class F, int CO>
__global__ void __launch_bounds__(256) tail64_tc32_kernel(const TailParams P) {
  using E = typename F::elem;
  constexpr int WT = 16 / CO;
  const int lane = threadIdx.x & 31;
  const int strips = (P.W + WT - 1) / WT, chunks = (P.H + TL_RC - 1) / TL_RC;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)P.B * strips * chunks) return;
  const int b = (int)(wid / (strips * chunks)), rem = (int)(wid - (long long)b * strips * chunks);
  const int r0 = (rem / strips) * TL_RC, xs = (rem % strips) * WT;
  // channel pair of this lane inside a pixel's 2 * 64 elements: block (2l) / CH, offset (2l) % CH; lo = hi + CH
  const int eo = ((2 * lane) / F::CH) * 2 * F::CH + (2 * lane) % F::CH;
  float w0[CO][9], w1[CO][9];
#pragma unroll
  for (int co = 0; co < CO; ++co)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const bool live = co < P.Cout;
      w0[co][t] = live ? __ldg(P.w + ((long long)co * 64 + 2 * lane) * 9 + t) : 0.f;
      w1[co][t] = live ? __ldg(P.w + ((long long)co * 64 + 2 * lane + 1) * 9 + t) : 0.f;
    }
  float acc[3][16];  // [output row slot][co * WT + j]
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[s][i] = 0.f;
  const bool poisoned = P.flag && *reinterpret_cast<const volatile int*>(P.flag) != 0;
  const E* img = static_cast<const E*>(P.x) + (long long)b * P.H * P.W * 128 + eo;
  const int tmax = min(TL_RC, P.H - r0) + 1;  // last input row index (t) that matters
  // the raw words of row t + 1 are requested before row t is converted and accumulated
  using RW = typename TailRaw<F>::type;
  RW ah[WT + 2], al[WT + 2], bh[WT + 2], bl[WT + 2];
  float c0[WT + 2], c1[WT + 2];
#define TL_LOAD(T, RH, RL) if ((T) <= tmax) tail_load_raw<F, WT>(img, r0 - 1 + (T), xs, P.H, P.W, RH, RL)
#define TL_ROW(PH, T, RH, RL)                                                                                                    \
  tail_convert<F, WT>((T) <= tmax && r0 - 1 + (T) >= 0 && r0 - 1 + (T) < P.H, xs, P.W, RH, RL, c0, c1);                          \
  tail_row<CO, PH>(P, T, tmax, b, r0, xs, lane, poisoned, w0, w1, acc, c0, c1)
  TL_LOAD(0, ah, al);
#pragma unroll 1
  for (int t = 0; t <= tmax; t += 6) {
    TL_LOAD(t + 1, bh, bl); TL_ROW(0, t, ah, al);
    TL_LOAD(t + 2, ah, al); TL_ROW(1, t + 1, bh, bl);
    TL_LOAD(t + 3, bh, bl); TL_ROW(2, t + 2, ah, al);
    TL_LOAD(t + 4, ah, al); TL_ROW(0, t + 3, bh, bl);
    TL_LOAD(t + 5, bh, bl); TL_ROW(1, t + 4, ah, al);
    TL_LOAD(t + 6, ah, al); TL_ROW(2, t + 5, bh, bl);
  }
#undef TL_LOAD
#undef TL_ROW
}

// split layout -> NCHW fp32 (tests / debugging): out[b,c,y,x] = hi + lo
template <class F>
__global__ void __launch_bounds__(256) split_to_nchw_kernel(const typename F::elem* __restrict__ in, float* __restrict__ out, int C, int H, int W,
                                                            long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long HW = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long pix = i / C;
    const int c = (int)(i - pix * C);
    const long long b = pix / HW, hw = pix - b * HW;
    const typename F::elem* s = in + pix * C * 2 + (c / F::CH) * 2 * F::CH + (c % F::CH);
    out[(b * C + c) * HW + hw] = (float)s[0] + (float)s[F::CH] * F::CORR;
  }
}
// NCHW fp32 -> split layout
template <class F>
__global__ void __launch_bounds__(256) nchw_to_split_kernel(const float* __restrict__ in, typename F::elem* __restrict__ out, int C, int H, int W,
                                                            long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long HW = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long pix = i / C;
    const int c = (int)(i - pix * C);
    const long long b = pix / HW, hw = pix - b * HW;
    const float v = __ldg(in + (b * C + c) * HW + hw);
    typename F::elem* d = out + pix * C * 2 + (c / F::CH) * 2 * F::CH + (c % F::CH);
    if constexpr (F::ID == 0) {
      const float hi = rna_tf32(v);
      d[0] = hi;
      d[F::CH] = v - hi;
    } else {
      const __half hi = __float2half_rn(v);
      d[0] = hi;
      d[F::CH] = __float2half_rn((v - __half2float(hi)) * 2048.0f);
    }
  }
}

#ifndef DINVK_EMUL
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

// 4-D activation view (words, X, Y, B) of a split16 tensor with arbitrary pixel strides (bytes)
template <class F>
static int make_act_map(CUtensorMap* m, const void* ptr, int B, int Y, int X, int C, long long sx, long long sy, long long sb, int box_x,
                        int box_y) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C * 2, (cuuint64_t)X, (cuuint64_t)Y, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)sx, (cuuint64_t)sy, (cuuint64_t)sb};
  cuuint32_t box[4] = {(cuuint32_t)(2 * F::CH), (cuuint32_t)box_x, (cuuint32_t)box_y, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, F::TM, 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(tc32 activations) failed: %d", (int)r);
  return 0;
}
template <class F>
static int make_w_map(CUtensorMap* m, const void* ptr, long long K, long long rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled is unavailable");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * F::EB};
  cuuint32_t box[2] = {(cuuint32_t)(2 * F::CH), 128};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, F::TM, 2, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(DINVK_ECUDA, "cuTensorMapEncodeTiled(tc32 weights) failed: %d", (int)r);
  return 0;
}

static int default_window() {
  static int w = -1;
  if (w < 0) {
    const char* e = getenv("DINVK_TC32_WINDOW");
    w = e ? std::max(1, atoi(e)) : 4;
  }
  return w;
}

template <class F>
static int launch(const Maps& M, const Params& P, void* stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc32_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(conv_tc32): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const long long tiles = (long long)P.B * P.tiles_y * P.tiles_x * P.n_tiles;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  count_launch();
  conv_tc32_kernel<F><<<grid, THREADS, SMEM, (cudaStream_t)stream>>>(M, P);
  return DINVK_POST_LAUNCH();
}

template <class F, int MH>
static int launch_slab(const Maps& M, const Params& P, void* stream) {
  using G = slab::Geom<MH>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc32_slab_kernel<F, MH>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::SMEM_BYTES);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "cudaFuncSetAttribute(conv_tc32_slab): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const long long tiles = (long long)P.B * P.tiles_y * P.tiles_x * P.n_tiles;
  const int grid = (int)std::min<long long>(tiles, sm_count());
  count_launch();
  conv_tc32_slab_kernel<F, MH><<<grid, G::THREADS, G::SMEM_BYTES, (cudaStream_t)stream>>>(M, P);
  return DINVK_POST_LAUNCH();
}

// kind 0: 3x3 stride 1 zero-pad 1 (weight rows = Cout/64 tiles of 128, K = 9*Cin, k = (ky*3+kx)*Cin + c)
// kind 1: 2x2 stride 2 (K = 4*Cin, k = (dy*2+dx)*Cin + c), out (B, H/2, W/2, Cout)
// kind 2: transposed 2x2 stride 2 (K = Cin, GEMM column = (dy*2+dx)*Cout + co), out (B, 2H, 2W, Cout)
template <class F>
static int conv_generic(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out, int B, int H,
                        int W, int Cin, int Cout, int kind, int act, int window, int* flag, void* stream) {
  DINVK_CHECK_ARG(x && weight && out, "conv_tc32: null pointer");
  DINVK_CHECK_ARG(B >= 0 && H >= 1 && W >= 1, "conv_tc32: bad shape");
  DINVK_CHECK_ARG(kind >= 0 && kind <= 2, "conv_tc32: kind=%d not in 0..2", kind);
  DINVK_CHECK_ARG(Cin % (2 * F::CH) == 0 && Cin >= 2 * F::CH, "conv_tc32: Cin=%d must be a multiple of %d", Cin, 2 * F::CH);
  DINVK_CHECK_ARG(Cout % 64 == 0 && Cout >= 64, "conv_tc32: Cout=%d must be a multiple of 64", Cout);
  DINVK_CHECK_ARG(kind != 1 || (H % 2 == 0 && W % 2 == 0), "conv_tc32: 2x2 stride-2 needs even H, W");
  DINVK_CHECK_ARG(kind == 0 || (!res && !res2), "conv_tc32: residual inputs are for kind 0 only");
  if (B == 0) return DINVK_OK;
  Maps M;
  Params P;
  int rc;
  const long long px = (long long)Cin * 2 * F::EB;  // bytes per input pixel
  P.B = B; P.Cin = Cin; P.Cout = Cout;
  P.kc_per_tap = Cin / (2 * F::CH);
  P.relu = act; P.res = res; P.res2 = res2; P.out = out; P.bias = bias; P.flag = flag;
  P.win = window > 0 ? window : default_window();
  for (int t = 0; t < 9; ++t) { P.dx[t] = 0; P.dy[t] = 0; P.amap[t] = 0; }
  if (kind == 0) {
    if ((rc = make_act_map<F>(&M.a[0], x, B, H, W, Cin, px, px * W, px * W * H, TX, TY))) return rc;
    M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
    if ((rc = make_w_map<F>(&M.b, weight, 9LL * Cin, 2LL * Cout))) return rc;
    P.H = H; P.W = W; P.ntaps = 9; P.mode = 0; P.n_tiles = Cout / 64;
    for (int t = 0; t < 9; ++t) { P.dx[t] = t % 3 - 1; P.dy[t] = t / 3 - 1; }
  } else if (kind == 1) {
    const int Ho = H / 2, Wo = W / 2;
    for (int t = 0; t < 4; ++t) {
      const char* base = reinterpret_cast<const char*>(x) + ((long long)(t >> 1) * W + (t & 1)) * px;
      if ((rc = make_act_map<F>(&M.a[t], base, B, Ho, Wo, Cin, 2 * px, 2 * px * W, px * W * H, TX, TY))) return rc;
      P.amap[t] = t;
    }
    if ((rc = make_w_map<F>(&M.b, weight, 4LL * Cin, 2LL * Cout))) return rc;
    P.H = Ho; P.W = Wo; P.ntaps = 4; P.mode = 0; P.n_tiles = Cout / 64;
  } else {
    if ((rc = make_act_map<F>(&M.a[0], x, B, H, W, Cin, px, px * W, px * W * H, TX, TY))) return rc;
    M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
    if ((rc = make_w_map<F>(&M.b, weight, (long long)Cin, 8LL * Cout))) return rc;
    P.H = H; P.W = W; P.ntaps = 1; P.mode = 2; P.n_tiles = 4 * Cout / 64;
  }
  P.tiles_x = ceil_div(P.W, TX); P.tiles_y = ceil_div(P.H, TY);
  // every 2x2 layer gains from sharing the activation tile between its N tiles (down 64 -> 128: 402 -> 297 us, up 256 -> 128: 415 -> 263 us):
  // with the N tile outermost each activation byte crossed HBM n_tiles (2 .. 8) times
  P.ngrp = getenv("DINVK_TC32_NT_OUTER") ? 1 : P.n_tiles;
  return launch<F>(M, P, stream);
}

// x-halves of the slab kernel's CTA tile: 1 = 8 x 16 pixels, two consumer warpgroups.  (With 2, four warpgroups of 64
// accumulator + 32 drain registers each do not fit the register file and spill.)
constexpr int SLAB_MH = 1;

template <class F>
static int conv_slab(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out, int B, int H, int W,
                     int Cin, int Cout, int act, int window, int* flag, void* stream) {
  DINVK_CHECK_ARG(x && weight && out, "conv_tc32_slab: null pointer");
  DINVK_CHECK_ARG(B >= 0 && H >= 1 && W >= 1, "conv_tc32_slab: bad shape");
  DINVK_CHECK_ARG(Cin % F::CH == 0 && Cin >= F::CH, "conv_tc32_slab: Cin=%d must be a multiple of %d", Cin, F::CH);
  DINVK_CHECK_ARG(Cout % 64 == 0 && Cout >= 64, "conv_tc32_slab: Cout=%d must be a multiple of 64", Cout);
  if (B == 0) return DINVK_OK;
  Maps M;
  Params P;
  int rc;
  const long long px = (long long)Cin * 2 * F::EB;
  using G = slab::Geom<SLAB_MH>;
  if ((rc = make_act_map<F>(&M.a[0], x, B, H, W, Cin, px, px * W, px * W * H, G::SLAB_X, slab::SLAB_Y))) return rc;
  M.a[1] = M.a[0]; M.a[2] = M.a[0]; M.a[3] = M.a[0];
  if ((rc = make_w_map<F>(&M.b, weight, 10LL * Cin, 2LL * Cout))) return rc;
  P.B = B; P.H = H; P.W = W; P.Cin = Cin; P.Cout = Cout;
  P.ntaps = 9; P.kc_per_tap = Cin / F::CH; P.mode = 0; P.n_tiles = Cout / 64;
  for (int t = 0; t < 9; ++t) { P.dx[t] = t % 3 - 1; P.dy[t] = t / 3 - 1; P.amap[t] = 0; }
  P.relu = act; P.res = res; P.res2 = res2; P.out = out; P.bias = bias; P.flag = flag;
  // accumulation window in channel blocks: ONE block by default = 18 full-scale accumulations (tf32: k = 144, fp16: k = 288),
  // so that the tensor core's own fp32 accumulation only ever sees short partial sums (DESIGN §4.4)
  static const int def_win = getenv("DINVK_TC32_SLAB_WINDOW") ? std::max(1, atoi(getenv("DINVK_TC32_SLAB_WINDOW"))) : 1;
  P.win = window > 0 ? window : def_win;
  P.tiles_x = ceil_div(W, G::TXP); P.tiles_y = ceil_div(H, slab::TYP);
  // N tiles of a pixel tile are adjacent work items in groups of at most 2, so that CTAs sharing a slab run together while
  // only one weight group at a time is streamed (DINVK_TC32_NT_GROUP overrides: 1 = N tile outermost)
  {
    static const int env_g = getenv("DINVK_TC32_NT_GROUP") ? atoi(getenv("DINVK_TC32_NT_GROUP")) : 0;
    int g = env_g > 0 ? env_g : (P.n_tiles <= 2 ? P.n_tiles : 1);
    while (g > 1 && P.n_tiles % g) --g;
    P.ngrp = std::max(1, std::min(g, P.n_tiles));
  }
  return launch_slab<F, SLAB_MH>(M, P, stream);
}

#endif  // !DINVK_EMUL
template <class F>
static int conv_head(const float* x_nchw, const float* weight, const float* bias, void* out, int B, int C, int H, int W, int Cout,
                     float fill_scalar, const float* fill_batch, int has_fill, int act, int* flag, void* stream) {
  const int CT = C + (has_fill ? 1 : 0);
  DINVK_CHECK_ARG(Cout % F::CH == 0 && Cout >= F::CH && Cout <= 256, "conv_tc32_head: Cout=%d must be a multiple of %d (<= 256)", Cout, F::CH);
  HeadParams P{x_nchw, weight, bias, out, B, C, H, W, Cout, fill_scalar, fill_batch, has_fill, act, flag};
  const long long npix = (long long)B * H * W;
  static const bool old_head = getenv("DINVK_TC32_OLD_HEAD") != nullptr;
  if (Cout == 64 && CT >= 1 && CT <= 4 && !old_head) {
    const long long warps = (long long)B * ceil_div(H, 2) * ceil_div(W, 32);
    const unsigned g = (unsigned)((warps + 7) / 8);
    switch (CT) {
      case 1: DINVK_LAUNCH((head64_tc32_kernel<F, 1>), dim3(g), dim3(256), 0, stream, P); break;
      case 2: DINVK_LAUNCH((head64_tc32_kernel<F, 2>), dim3(g), dim3(256), 0, stream, P); break;
      case 3: DINVK_LAUNCH((head64_tc32_kernel<F, 3>), dim3(g), dim3(256), 0, stream, P); break;
      default: DINVK_LAUNCH((head64_tc32_kernel<F, 4>), dim3(g), dim3(256), 0, stream, P); break;
    }
    return DINVK_POST_LAUNCH();
  }
  const unsigned grid = (unsigned)((npix + 255) / 256);
  const size_t smem = (size_t)Cout * ((9 * CT + 3) & ~3) * 4;
  switch (CT) {
    case 1: DINVK_LAUNCH((head_tc32_kernel<F, 1>), dim3(grid), dim3(256), smem, stream, P); break;
    case 2: DINVK_LAUNCH((head_tc32_kernel<F, 2>), dim3(grid), dim3(256), smem, stream, P); break;
    case 3: DINVK_LAUNCH((head_tc32_kernel<F, 3>), dim3(grid), dim3(256), smem, stream, P); break;
    default: DINVK_LAUNCH((head_tc32_kernel<F, 4>), dim3(grid), dim3(256), smem, stream, P); break;
  }
  return DINVK_POST_LAUNCH();
}

template <class F>
static int conv_tail(const void* x, const float* weight, const float* bias, const float* add_nchw, float* out_nchw, int B, int H, int W,
                     int Cin, int Cout, const int* flag, void* stream) {
  DINVK_CHECK_ARG(Cin % F::CH == 0 && Cin >= F::CH && Cin <= 128, "conv_tc32_tail: Cin=%d must be a multiple of %d (<= 128)", Cin, F::CH);
  TailParams P{x, weight, bias, add_nchw, out_nchw, B, H, W, Cin, Cout, flag};
  static const bool old_tail = getenv("DINVK_TC32_OLD_TAIL") != nullptr;
  if (Cin == 64 && Cout >= 1 && Cout <= 4 && !old_tail) {
    const int co = Cout == 3 ? 4 : Cout, wt = 16 / co;
    const long long warps = (long long)B * ceil_div(W, wt) * ceil_div(H, TL_RC);
    const unsigned grid = (unsigned)((warps + 7) / 8);
    if (co == 1) DINVK_LAUNCH((tail64_tc32_kernel<F, 1>), dim3(grid), dim3(256), 0, stream, P);
    else if (co == 2) DINVK_LAUNCH((tail64_tc32_kernel<F, 2>), dim3(grid), dim3(256), 0, stream, P);
    else DINVK_LAUNCH((tail64_tc32_kernel<F, 4>), dim3(grid), dim3(256), 0, stream, P);
    return DINVK_POST_LAUNCH();
  }
  const int tiles = B * ceil_div(H, TL_TY) * ceil_div(W, TL_TX);
  const int CO = Cout <= 2 ? 2 : 4;
  const size_t smem = ((size_t)(TL_TY + 2) * (TL_TX + 2) * (Cin + 4) + (size_t)CO * 9 * Cin) * 4;
  int rc;
  if (CO == 2) {
    if ((rc = allow_smem(tail_tc32_kernel<F, 2>, smem))) return rc;
    DINVK_LAUNCH((tail_tc32_kernel<F, 2>), dim3(tiles), dim3(256), smem, stream, P);
  } else {
    if ((rc = allow_smem(tail_tc32_kernel<F, 4>, smem))) return rc;
    DINVK_LAUNCH((tail_tc32_kernel<F, 4>), dim3(tiles), dim3(256), smem, stream, P);
  }
  return DINVK_POST_LAUNCH();
}

}  // namespace t32
}  // namespace dinvk

using namespace dinvk;

#define DINVK_FMT_DISPATCH(fmt, call_tf32, call_f16)                                                   \
  do {                                                                                                 \
    if ((fmt) == 0) return call_tf32;                                                                  \
    if ((fmt) == 1) return call_f16;                                                                   \
    return ::dinvk::set_error(DINVK_EINVAL, "conv_tc32: fmt=%d not in {0 (tf32 split16), 1 (fp16 split32)}", (fmt)); \
  } while (0)

#ifndef DINVK_EMUL
extern "C" int dinvk_conv_tc32(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out, int B,
                               int H, int W, int Cin, int Cout, int kind, int act, int window, int fmt, int* overflow_flag, void* stream) {
  using namespace t32;
  DINVK_FMT_DISPATCH(fmt, conv_generic<FmtTF32>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, kind, act, window, overflow_flag, stream),
                     conv_generic<FmtF16>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, kind, act, window, overflow_flag, stream));
}

extern "C" int dinvk_conv_tc32_slab(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                                    int B, int H, int W, int Cin, int Cout, int act, int window, int fmt, int* overflow_flag,
                                    void* stream) {
  using namespace t32;
  DINVK_FMT_DISPATCH(fmt, conv_slab<FmtTF32>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, act, window, overflow_flag, stream),
                     conv_slab<FmtF16>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, act, window, overflow_flag, stream));
}

#endif  // !DINVK_EMUL
extern "C" int dinvk_conv_tc32_head(const float* x_nchw, const float* weight, const float* bias, void* out, int B, int C, int H, int W,
                                    int Cout, float fill_scalar, const float* fill_batch, int has_fill, int act, int fmt,
                                    int* overflow_flag, void* stream) {
  using namespace t32;
  DINVK_CHECK_ARG(x_nchw && weight && out && B >= 0 && C >= 1 && H >= 1 && W >= 1, "conv_tc32_head: bad arguments");
  const int CT = C + (has_fill ? 1 : 0);
  DINVK_CHECK_ARG(CT >= 1 && CT <= 4, "conv_tc32_head: %d input channels (incl. noise map) not in 1..4", CT);
  if (B == 0) return DINVK_OK;
  DINVK_FMT_DISPATCH(fmt, conv_head<FmtTF32>(x_nchw, weight, bias, out, B, C, H, W, Cout, fill_scalar, fill_batch, has_fill, act, overflow_flag, stream),
                     conv_head<FmtF16>(x_nchw, weight, bias, out, B, C, H, W, Cout, fill_scalar, fill_batch, has_fill, act, overflow_flag, stream));
}

extern "C" int dinvk_conv_tc32_tail(const void* x, const float* weight, const float* bias, const float* add_nchw, float* out_nchw, int B,
                                    int H, int W, int Cin, int Cout, int fmt, const int* overflow_flag, void* stream) {
  using namespace t32;
  DINVK_CHECK_ARG(x && weight && out_nchw && B >= 0 && H >= 1 && W >= 1, "conv_tc32_tail: bad arguments");
  DINVK_CHECK_ARG(Cout >= 1 && Cout <= 4, "conv_tc32_tail: Cout=%d not in 1..4", Cout);
  if (B == 0) return DINVK_OK;
  DINVK_FMT_DISPATCH(fmt, conv_tail<FmtTF32>(x, weight, bias, add_nchw, out_nchw, B, H, W, Cin, Cout, overflow_flag, stream),
                     conv_tail<FmtF16>(x, weight, bias, add_nchw, out_nchw, B, H, W, Cin, Cout, overflow_flag, stream));
}

template <class F>
static int split_convert(const void* in, void* out, int B, int C, int H, int W, int to_nchw, void* stream) {
  using namespace t32;
  DINVK_CHECK_ARG(in && out && B >= 0 && C % F::CH == 0 && C >= F::CH, "split converter: C=%d must be a multiple of %d", C, F::CH);
  if (B == 0) return DINVK_OK;
  const long long n = (long long)B * H * W * C;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sm_count() * 16);
  if (to_nchw) {
    DINVK_LAUNCH(split_to_nchw_kernel<F>, dim3(grid), dim3(256), 0, stream, static_cast<const typename F::elem*>(in), static_cast<float*>(out), C, H, W, n);
  } else {
    DINVK_LAUNCH(nchw_to_split_kernel<F>, dim3(grid), dim3(256), 0, stream, static_cast<const float*>(in), static_cast<typename F::elem*>(out), C, H, W, n);
  }
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_split16_to_nchw(const void* in, float* out, int B, int C, int H, int W, int fmt, void* stream) {
  DINVK_FMT_DISPATCH(fmt, split_convert<t32::FmtTF32>(in, out, B, C, H, W, 1, stream), split_convert<t32::FmtF16>(in, out, B, C, H, W, 1, stream));
}

extern "C" int dinvk_nchw_to_split16(const float* in, void* out, int B, int C, int H, int W, int fmt, void* stream) {
  DINVK_FMT_DISPATCH(fmt, split_convert<t32::FmtTF32>(in, out, B, C, H, W, 0, stream), split_convert<t32::FmtF16>(in, out, B, C, H, W, 0, stream));
}
