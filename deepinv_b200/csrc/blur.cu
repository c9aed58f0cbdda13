// blur.cu — direct (im2col-free) 2-D convolution for Blur.A / Blur.A_adjoint, all five paddings.
//
// Replaces deepinv/physics/functional/convolution.py:42-164 (conv2d / conv_transpose2d: flip + F.pad +
// grouped F.conv2d, and F.conv_transpose2d + _apply_transpose_padding :641-758) for the reference's
// per-sample / per-channel filter broadcast (:761-787).
//
// Everything is one tiled correlation kernel
//     out[i,j] = sum_{u,v} ks[u,v] * in[ map(i + u + off_i), map(j + v + off_j) ]
// where ks is the filter staged in shared memory (flipped for a true convolution), `map` resolves the
// padding rule in index space (zeros / circular / replicate / reflect) while the input tile + halo is
// staged, and (off_i, off_j) place the kernel origin:
//     A,  same-size paddings : flip, off = h/2 - (h-1),           map = padding rule, out (H, W)
//     A,  valid              : flip, off = 0,                      no map,             out (H-h+1, W-w+1)
//     A^T valid              : no flip, off = -(h-1), zeros,       in (H-h+1, W-w+1),  out (H, W)
//     A^T circular/constant  : no flip, off = -h/2, circular/zeros                     out (H, W)
//     A^T replicate/reflect  : no flip, off = -(h-1), zeros -> extended (H+h-1, W+w-1) image, then the
//                              transpose of the padding folds the border strips back (fold kernel).
// A CTA computes a 64x64 output tile; each thread owns 4x4 outputs and slides a 4-wide register window
// along the filter row (one 128-bit shared load per 16 FMAs per row).  Filters up to 123x123 fit (200 KB of shared memory).
//
// The space-varying blur (product convolution, SpaceVaryingBlur) runs the same tile and window loop K times per CTA, once per
// term, into one set of accumulators: svblur_fwd_kernel on the product patch w_k . x, svblur_adj_kernel on the y patch with a
// per-pixel multiplier applied to each term's partial block.  The replicate / reflect adjoint folds once, after the K terms.
#include "common.cuh"
#include "tma_tile.cuh"

#include <algorithm>
#include <cstdlib>

namespace dinvk {

constexpr int BL_T = 64;  // tile edge

struct BlurParams {
  int C, Hin, Win, Hout, Wout, h, w, wp;  // wp = w rounded up to a multiple of 4
  int FB, FC, flip, off_i, off_j, map;    // map: 0 zeros, 1 circular, 2 replicate, 3 reflect
  int PW;                                 // patch row pitch (floats)
  int shift;                              // zero taps prepended to every filter row (0..3): makes off_j a multiple of 4
  int tiles_x;
};

__device__ __forceinline__ int map_index(int a, int n, int mode, bool& ok) {
  ok = true;
  if (mode == 1) { a %= n; return a < 0 ? a + n : a; }
  if (mode == 2) return a < 0 ? 0 : (a >= n ? n - 1 : a);
  if (mode == 3) { if (a < 0) a = -a; if (a > n - 1) a = 2 * (n - 1) - a; ok = (a >= 0 && a < n); return ok ? a : 0; }
  ok = (a >= 0 && a < n);
  return ok ? a : 0;
}

// Helpers of the space-varying kernels below: the staging and window loop of blur_corr_kernel, factored out.  blur_corr_kernel
// keeps its own inline copy so that its code generation stays exactly as it was.
//
// the filter of one term, staged as the window loop reads it: ks[u][v] for v < wp, `shift` leading zero taps (see corr_params)
__device__ __forceinline__ void stage_filter(float* ks, const float* __restrict__ f, const BlurParams& P) {
  for (int idx = threadIdx.x; idx < P.h * P.wp; idx += 256) {
    const int u = idx / P.wp, v = idx - u * P.wp - P.shift;
    float val = 0.f;
    if (v >= 0 && v < P.w) val = P.flip ? __ldg(f + (P.h - 1 - u) * P.w + (P.w - 1 - v)) : __ldg(f + u * P.w + v);
    ks[idx] = val;
  }
}

// The input tile + halo of plane `bc`, rows i0 + off_i.., columns j0 + off_j...  Zero padding (and every tile whose halo stays inside
// the image, whatever the padding rule) is ONE tensor-map box load: the copy engine zero-fills out-of-range elements.  Tiles that
// touch the border under circular / replicate / reflect padding resolve the rule in index space with the cooperative loop.
// No barrier at the end: the caller's __syncthreads publishes the patch.
__device__ __forceinline__ void stage_patch(float* patch, const tt::TileMap* tmap, int use_tma, const float* __restrict__ src,
                                            const BlurParams& P, int i0, int j0, int bc) {
  const int PH = BL_T + P.h - 1;
  bool by_tma = false;
#ifndef DINVK_EMUL
  if (use_tma) {
    const int r0 = i0 + P.off_i, c0 = j0 + P.off_j;
    by_tma = (P.map == 0) || (r0 >= 0 && r0 + PH <= P.Hin && c0 >= 0 && c0 + P.PW <= P.Win);
    if (by_tma) {   // (uniform over the CTA)
      __shared__ __align__(8) uint64_t tile_bar;
      tt::stage_tile(patch, tmap, &tile_bar, c0, r0, bc, (uint32_t)(PH * P.PW * 4));
    }
  }
#else
  (void)tmap; (void)use_tma; (void)bc;
#endif
  if (!by_tma) {
    for (int idx = threadIdx.x; idx < PH * P.PW; idx += 256) {
      const int pr = idx / P.PW, pc = idx - pr * P.PW;
      bool okr, okc;
      const int gi = map_index(i0 + pr + P.off_i, P.Hin, P.map, okr);
      const int gj = map_index(j0 + pc + P.off_j, P.Win, P.map, okc);
      patch[idx] = (okr && okc) ? __ldg(src + (long long)gi * P.Win + gj) : 0.f;
    }
  }
}

// the 4x4 register-tiled sliding window: acc[r][q] += sum_{u,v} ks[u][v] * patch[ty*4 + r + u][tx*4 + q + v], one 128-bit shared
// load per 16 FMAs per filter row
__device__ __forceinline__ void window_fma(const float* patch, const float* ks, const BlurParams& P, int tx, int ty, float (&acc)[4][4]) {
  const int nchunk = P.wp >> 2;
  for (int u = 0; u < P.h; ++u) {
    float4 lo[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) lo[r] = *reinterpret_cast<const float4*>(&patch[(ty * 4 + r + u) * P.PW + tx * 4]);
    const float4* krow = reinterpret_cast<const float4*>(&ks[u * P.wp]);
    for (int vb = 0; vb < nchunk; ++vb) {
      const float4 k4 = krow[vb];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 hi = *reinterpret_cast<const float4*>(&patch[(ty * 4 + r + u) * P.PW + tx * 4 + 4 * vb + 4]);
        const float win[8] = {lo[r].x, lo[r].y, lo[r].z, lo[r].w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float a = acc[r][q];
          a = fmaf(k4.x, win[q], a);
          a = fmaf(k4.y, win[q + 1], a);
          a = fmaf(k4.z, win[q + 2], a);
          a = fmaf(k4.w, win[q + 3], a);
          acc[r][q] = a;
        }
        lo[r] = hi;
      }
    }
  }
}

__device__ __forceinline__ float* align128(float* p) {
  return reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(p) + 127) & ~static_cast<uintptr_t>(127));
}

__device__ __forceinline__ void store_tile(float* __restrict__ dst, const float (&acc)[4][4], const BlurParams& P, int i0, int j0,
                                           int tx, int ty) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int gi = i0 + ty * 4 + r;
    if (gi >= P.Hout) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int gj = j0 + tx * 4 + q;
      if (gj < P.Wout) dst[(long long)gi * P.Wout + gj] = acc[r][q];
    }
  }
}

__global__ void __launch_bounds__(256) blur_corr_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                        const float* __restrict__ in, const float* __restrict__ filt,
                                                        float* __restrict__ out, BlurParams P) {
  DINVK_DYN_SMEM(float, smem);
  float* ks = smem;                 // [h][wp]
  // [(BL_T + h - 1)][PW], 128-byte aligned at run time (TMA destination; the launch reserves the slack)
  float* patch = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(smem + P.h * P.wp) + 127) & ~static_cast<uintptr_t>(127));
  const int tid = threadIdx.x;
  const int bc = blockIdx.y;
  const int b = bc / P.C, c = bc - b * P.C;
  const int i0 = (blockIdx.x / P.tiles_x) * BL_T, j0 = (blockIdx.x % P.tiles_x) * BL_T;
  const float* f = filt + ((long long)(P.FB == 1 ? 0 : b) * P.FC + (P.FC == 1 ? 0 : c)) * P.h * P.w;
  for (int idx = tid; idx < P.h * P.wp; idx += 256) {
    const int u = idx / P.wp, v = idx - u * P.wp - P.shift;   // `shift` leading zero taps: see launch_corr
    float val = 0.f;
    if (v >= 0 && v < P.w) val = P.flip ? __ldg(f + (P.h - 1 - u) * P.w + (P.w - 1 - v)) : __ldg(f + u * P.w + v);
    ks[idx] = val;
  }
  const int PH = BL_T + P.h - 1;
  const float* src = in + (long long)bc * P.Hin * P.Win;
  // The input tile + halo.  Zero padding (and every tile whose halo stays inside the image, whatever the padding rule) is ONE
  // tensor-map box load: the copy engine zero-fills out-of-range elements.  Tiles that touch the border under circular /
  // replicate / reflect padding resolve the rule in index space with the cooperative loop.
  bool by_tma = false;
#ifndef DINVK_EMUL
  if (use_tma) {
    const int r0 = i0 + P.off_i, c0 = j0 + P.off_j;
    by_tma = (P.map == 0) || (r0 >= 0 && r0 + PH <= P.Hin && c0 >= 0 && c0 + P.PW <= P.Win);
    if (by_tma) {   // (uniform over the CTA)
      __shared__ __align__(8) uint64_t tile_bar;
      tt::stage_tile(patch, &tmap, &tile_bar, c0, r0, bc, (uint32_t)(PH * P.PW * 4));
    }
  }
#endif
  if (!by_tma) {
    for (int idx = tid; idx < PH * P.PW; idx += 256) {
      const int pr = idx / P.PW, pc = idx - pr * P.PW;
      bool okr, okc;
      const int gi = map_index(i0 + pr + P.off_i, P.Hin, P.map, okr);
      const int gj = map_index(j0 + pc + P.off_j, P.Win, P.map, okc);
      patch[idx] = (okr && okc) ? __ldg(src + (long long)gi * P.Win + gj) : 0.f;
    }
  }
  __syncthreads();

  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
  const int nchunk = P.wp >> 2;
  for (int u = 0; u < P.h; ++u) {
    float4 lo[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) lo[r] = *reinterpret_cast<const float4*>(&patch[(ty * 4 + r + u) * P.PW + tx * 4]);
    const float4* krow = reinterpret_cast<const float4*>(&ks[u * P.wp]);
    for (int vb = 0; vb < nchunk; ++vb) {
      const float4 k4 = krow[vb];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 hi = *reinterpret_cast<const float4*>(&patch[(ty * 4 + r + u) * P.PW + tx * 4 + 4 * vb + 4]);
        const float win[8] = {lo[r].x, lo[r].y, lo[r].z, lo[r].w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float a = acc[r][q];
          a = fmaf(k4.x, win[q], a);
          a = fmaf(k4.y, win[q + 1], a);
          a = fmaf(k4.z, win[q + 2], a);
          a = fmaf(k4.w, win[q + 3], a);
          acc[r][q] = a;
        }
        lo[r] = hi;
      }
    }
  }
  // The window loop also runs the zero taps (the `shift` leading ones and the pad to wp) against real patch values, and 0 * NaN =
  // 0 * Inf = NaN: a non-finite pixel would reach up to 8 columns instead of its w-column footprint.  Such a zero tap adds 0 *
  // finite = +-0 to every other output, so only a non-finite accumulator can carry the leak; it is recomputed from the real taps
  // v in [shift, shift + w), in the loop's u-major order (the patch and filter stay resident: no barrier).  One rolled loop over
  // the flagged outputs: a repair unrolled per output took 66 registers, this form 48 (sm_90a), 0 spills.
  unsigned bad = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) bad |= (unsigned)((__float_as_uint(acc[r][q]) & 0x7f800000u) == 0x7f800000u) << (4 * r + q);
#pragma unroll 1
  for (int e = 0; bad >> e; ++e) {
    if (!((bad >> e) & 1)) continue;
    const float* prow = &patch[(ty * 4 + (e >> 2)) * P.PW + tx * 4 + (e & 3)];
    float a = 0.f;
    for (int u = 0; u < P.h; ++u)
      for (int v = P.shift; v < P.shift + P.w; ++v) a = fmaf(ks[u * P.wp + v], prow[u * P.PW + v], a);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (4 * r + q == e) acc[r][q] = a;
  }
  float* dst = out + (long long)bc * P.Hout * P.Wout;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int gi = i0 + ty * 4 + r;
    if (gi >= P.Hout) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int gj = j0 + tx * 4 + q;
      if (gj < P.Wout) dst[(long long)gi * P.Wout + gj] = acc[r][q];
    }
  }
}

// ---- space-varying blur (product convolution) -------------------------------------------------------------------------------
// A x = sum_k h_k * (w_k . x): each term is the correlation above run on the product patch, all K terms into the same
// accumulators.  Multipliers (MB, MC, K, H, W) and filters (FB, FC, K, h, w) broadcast independently over (B, C).
struct SvParams {
  BlurParams P;              // one term's geometry, exactly as blur_corr_kernel runs it
  int K, MB, MC;
  int woff_i, woff_j, wmap;  // adjoint: output pixel (i, j) takes the multiplier w[map(i + woff_i)][map(j + woff_j)] (H x W plane)
  int Hm, Wm;                // multiplier plane
  int xs;                    // forward: 1 = the x patch is staged once in shared memory, 0 = x is re-read through L1 / L2 for every k
};

// Forward.  Per k: stage filter k (flipped) and the product patch w_k[map(e)] * x[map(e)] (the reference pads w_k . x, so a padded
// position holds exactly that product), then the window loop.  Shared memory: ks, the product patch, and (xs) the x patch.
__global__ void __launch_bounds__(256, 2) svblur_fwd_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                         const float* __restrict__ x, const float* __restrict__ mult,
                                                         const float* __restrict__ filt, float* __restrict__ y, SvParams S) {
  const BlurParams& P = S.P;
  DINVK_DYN_SMEM(float, smem);
  const int PH = BL_T + P.h - 1;
  float* ks = smem;
  float* prod = align128(smem + P.h * P.wp);
  float* xp = align128(prod + PH * P.PW);
  const int tid = threadIdx.x;
  const int bc = blockIdx.y;
  const int b = bc / P.C, c = bc - b * P.C;
  const int i0 = (blockIdx.x / P.tiles_x) * BL_T, j0 = (blockIdx.x % P.tiles_x) * BL_T;
  const long long plane = (long long)P.Hin * P.Win;
  const float* src = x + (long long)bc * plane;
  const float* wb = mult + ((long long)(S.MB == 1 ? 0 : b) * S.MC + (S.MC == 1 ? 0 : c)) * S.K * plane;
  const float* fb = filt + ((long long)(P.FB == 1 ? 0 : b) * P.FC + (P.FC == 1 ? 0 : c)) * S.K * P.h * P.w;
  if (S.xs) stage_patch(xp, &tmap, use_tma, src, P, i0, j0, bc);

  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
  for (int k = 0; k < S.K; ++k) {
    __syncthreads();  // the window loop of term k - 1 is done with ks and prod (k = 0: the x patch has landed)
    stage_filter(ks, fb + (long long)k * P.h * P.w, P);
    const float* wk = wb + k * plane;
    for (int idx = tid; idx < PH * P.PW; idx += 256) {
      const int pr = idx / P.PW, pc = idx - pr * P.PW;
      bool okr, okc;
      const int gi = map_index(i0 + pr + P.off_i, P.Hin, P.map, okr);
      const int gj = map_index(j0 + pc + P.off_j, P.Win, P.map, okc);
      float v = 0.f;
      if (okr && okc) {
        const long long g = (long long)gi * P.Win + gj;
        v = (S.xs ? xp[idx] : __ldg(src + g)) * __ldg(wk + g);
      }
      prod[idx] = v;
    }
    __syncthreads();
    window_fma(prod, ks, P, tx, ty, acc);
  }
  store_tile(y + (long long)bc * P.Hout * P.Wout, acc, P, i0, j0, tx, ty);
}

// Adjoint.  The y patch is staged once; per k the correlation with the unflipped h_k goes into a partial block that is scaled by
// w_k at the output pixel and added to the totals.  On the extended (H+h-1, W+w-1) domain of replicate / reflect the output pixel e
// takes w_k[map(e)]: the fold sums the e with map(e) = p, over which w_k[p] is constant, so scaling before the fold is exact.
__global__ void __launch_bounds__(256) svblur_adj_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                         const float* __restrict__ yin, const float* __restrict__ mult,
                                                         const float* __restrict__ filt, float* __restrict__ out, SvParams S) {
  const BlurParams& P = S.P;
  DINVK_DYN_SMEM(float, smem);
  float* ks = smem;
  float* patch = align128(smem + P.h * P.wp);
  const int tid = threadIdx.x;
  const int bc = blockIdx.y;
  const int b = bc / P.C, c = bc - b * P.C;
  const int i0 = (blockIdx.x / P.tiles_x) * BL_T, j0 = (blockIdx.x % P.tiles_x) * BL_T;
  const long long mplane = (long long)S.Hm * S.Wm;
  const float* wb = mult + ((long long)(S.MB == 1 ? 0 : b) * S.MC + (S.MC == 1 ? 0 : c)) * S.K * mplane;
  const float* fb = filt + ((long long)(P.FB == 1 ? 0 : b) * P.FC + (P.FC == 1 ? 0 : c)) * S.K * P.h * P.w;
  stage_patch(patch, &tmap, use_tma, yin + (long long)bc * P.Hin * P.Win, P, i0, j0, bc);

  const int tx = tid & 15, ty = tid >> 4;
  int mi[4], mj[4];  // multiplier row / column of this thread's outputs (clamped to 0 past the output edge; never stored)
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    bool ok;
    mi[e] = map_index(i0 + ty * 4 + e + S.woff_i, S.Hm, S.wmap, ok);
    mj[e] = map_index(j0 + tx * 4 + e + S.woff_j, S.Wm, S.wmap, ok);
  }
  float tot[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) tot[r][q] = 0.f;
  for (int k = 0; k < S.K; ++k) {
    __syncthreads();  // the window loop of term k - 1 is done with ks
    stage_filter(ks, fb + (long long)k * P.h * P.w, P);
    __syncthreads();
    float part[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) part[r][q] = 0.f;
    window_fma(patch, ks, P, tx, ty, part);
    const float* wk = wb + k * mplane;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) tot[r][q] = fmaf(part[r][q], __ldg(wk + (long long)mi[r] * S.Wm + mj[q]), tot[r][q]);
  }
  store_tile(out + (long long)bc * P.Hout * P.Wout, tot, P, i0, j0, tx, ty);
}

// ---- tiled space-varying blur (tiled product convolution) -------------------------------------------------------------------
// A x = sum_k Wt_k . (h_k *valid x), A^T y = sum_k h_k (transposed valid) (Wt_k . y).  Patch k = r * nc + c covers rows
// [r s1, r s1 + P1) and columns [c s2, c s2 + P2) of the compatible grid, whose origin is x's; its multiplier w_k (P1 x P2, shared
// over B and C) is placed there, and Wt_k is that plane cropped to the valid output, which sits at (a_i, a_j) = (h/2, w/2).
// A tile visits only the (r, c) rectangle of patches that can reach it, never all K.  Tile t of the grid has origin G = 64 t in
// stage_patch's coordinates and stores outputs G - d.. (d_i, d_j below, rows and columns before 0 are masked): the forward uses
// d = a, so its tiles lie on multiples of 64 of the compatible grid (one stride cell per tile when the stride is a multiple of 64
// that divides the patch); the adjoint uses d = 32, which centres the tile's read span (64 + h - 1) on a multiple of 64.
struct TsvParams {
  BlurParams P;        // one term's geometry; Hout x Wout is the output plane
  int K, nr, nc, P1, P2, s1, s2;
  int ai, aj;          // compatible coordinates of y's origin
  int di, dj;          // output origin of tile G = G - d
  int Hy, Wy;          // y plane (the valid output)
  int xs;              // adjoint: 1 = the y patch is staged once in shared memory, 0 = y is re-read through L1 / L2 for every term
};

// patches [*lo, *hi] along one dimension whose span [n s, n s + p) meets the compatible interval [a, b]; empty when *lo > *hi
__device__ __forceinline__ void term_range(int a, int b, int p, int s, int n, int* lo, int* hi) {
  const int e = a - p + 1;  // span end must pass a
  *lo = e <= 0 ? 0 : (e + s - 1) / s;
  *hi = a > b ? -1 : min(n - 1, b / s);  // (a >= 0 here)
}

__device__ __forceinline__ void store_tile_masked(float* __restrict__ dst, const float (&acc)[4][4], const BlurParams& P, int i0,
                                                  int j0, int tx, int ty) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int gi = i0 + ty * 4 + r;
    if (gi < 0 || gi >= P.Hout) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int gj = j0 + tx * 4 + q;
      if (gj >= 0 && gj < P.Wout) dst[(long long)gi * P.Wout + gj] = acc[r][q];
    }
  }
}

// Forward.  The x patch is staged once; per term the correlation with the flipped h_k goes into a partial block, which is added
// times w_k at every output pixel inside patch k (and nowhere else: a non-finite h_k reaches exactly its footprint).  A warp (8
// output rows) skips the window loop of a term whose rows it does not meet.
__global__ void __launch_bounds__(256) tiled_svblur_fwd_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                               const float* __restrict__ x, const float* __restrict__ mult,
                                                               const float* __restrict__ filt, float* __restrict__ y, TsvParams S) {
  const BlurParams& P = S.P;
  DINVK_DYN_SMEM(float, smem);
  float* ks = smem;
  float* patch = align128(smem + P.h * P.wp);
  const int tid = threadIdx.x;
  const int bc = blockIdx.y;
  const int b = bc / P.C, c = bc - b * P.C;
  const int gi = (blockIdx.x / P.tiles_x) * BL_T, gj = (blockIdx.x % P.tiles_x) * BL_T;
  const int oi = gi - S.di, oj = gj - S.dj;  // output origin; compatible coordinates of the tile's outputs: o + a
  int r0, r1, c0, c1;
  term_range(max(oi, 0) + S.ai, min(oi + BL_T, P.Hout) - 1 + S.ai, S.P1, S.s1, S.nr, &r0, &r1);
  term_range(max(oj, 0) + S.aj, min(oj + BL_T, P.Wout) - 1 + S.aj, S.P2, S.s2, S.nc, &c0, &c1);
  if (r0 > r1 || c0 > c1) return;  // (uniform) a tile of masked outputs only
  const float* fb = filt + ((long long)(P.FB == 1 ? 0 : b) * P.FC + (P.FC == 1 ? 0 : c)) * S.K * P.h * P.w;
  stage_patch(patch, &tmap, use_tma, x + (long long)bc * P.Hin * P.Win, P, gi, gj, bc);

  const int tx = tid & 15, ty = tid >> 4;
  const int wr = oi + S.ai + (ty & ~1) * 4;  // first compatible row of this warp's outputs
  float tot[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) tot[r][q] = 0.f;
  for (int pr = r0; pr <= r1; ++pr) {
    for (int pc = c0; pc <= c1; ++pc) {
      const int k = pr * S.nc + pc;
      __syncthreads();  // the window loop of the previous term is done with ks
      stage_filter(ks, fb + (long long)k * P.h * P.w, P);
      __syncthreads();  // (first term: the x patch has landed as well)
      const int ri = oi + S.ai - pr * S.s1, rj = oj + S.aj - pc * S.s2;  // tile origin in patch k's multiplier plane
      if (wr + 8 <= pr * S.s1 || wr >= pr * S.s1 + S.P1) continue;  // (warp-uniform)
      float part[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) part[r][q] = 0.f;
      window_fma(patch, ks, P, tx, ty, part);
      const float* wk = mult + (long long)k * S.P1 * S.P2;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int I = ri + ty * 4 + r;
        if (I < 0 || I >= S.P1) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int J = rj + tx * 4 + q;
          if (J >= 0 && J < S.P2) tot[r][q] = fmaf(part[r][q], __ldg(wk + (long long)I * S.P2 + J), tot[r][q]);
        }
      }
    }
  }
  store_tile_masked(y + (long long)bc * P.Hout * P.Wout, tot, P, oi, oj, tx, ty);
}

// Adjoint.  Per term: stage the unflipped h_k and the product patch Wt_k . y (zero outside patch k and outside y), run the window
// loop into a partial block and add it at the output pixels within patch k's footprint grown by the filter (where a non-finite
// h_k reaches in the reference, and the only pixels a finite one can change).  A warp skips terms whose grown rows it does not meet.
__global__ void __launch_bounds__(256, 2) tiled_svblur_adj_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                                  const float* __restrict__ yin, const float* __restrict__ mult,
                                                                  const float* __restrict__ filt, float* __restrict__ out,
                                                                  TsvParams S) {
  const BlurParams& P = S.P;
  DINVK_DYN_SMEM(float, smem);
  const int PH = BL_T + P.h - 1;
  float* ks = smem;
  float* prod = align128(smem + P.h * P.wp);
  float* yp = align128(prod + PH * P.PW);
  const int tid = threadIdx.x;
  const int bc = blockIdx.y;
  const int b = bc / P.C, c = bc - b * P.C;
  const int gi = (blockIdx.x / P.tiles_x) * BL_T, gj = (blockIdx.x % P.tiles_x) * BL_T;
  const int oi = gi - S.di, oj = gj - S.dj;  // output origin (x coordinates = compatible coordinates)
  // output rows [lo, hi] read y rows [lo - (h - 1), hi] (cut to y), i.e. compatible rows + a
  int r0, r1, c0, c1;
  term_range(max(max(oi, 0) - (P.h - 1), 0) + S.ai, min(min(oi + BL_T, P.Hout) - 1, S.Hy - 1) + S.ai, S.P1, S.s1, S.nr, &r0, &r1);
  term_range(max(max(oj, 0) - (P.w - 1), 0) + S.aj, min(min(oj + BL_T, P.Wout) - 1, S.Wy - 1) + S.aj, S.P2, S.s2, S.nc, &c0, &c1);
  if (r0 > r1 || c0 > c1) return;  // (uniform) a tile of masked outputs only
  const float* fb = filt + ((long long)(P.FB == 1 ? 0 : b) * P.FC + (P.FC == 1 ? 0 : c)) * S.K * P.h * P.w;
  const float* src = yin + (long long)bc * P.Hin * P.Win;
  if (S.xs) stage_patch(yp, &tmap, use_tma, src, P, gi, gj, bc);

  const int tx = tid & 15, ty = tid >> 4;
  const int wr = oi + (ty & ~1) * 4;  // first output row of this warp
  float tot[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < 4; ++q) tot[r][q] = 0.f;
  for (int pr = r0; pr <= r1; ++pr) {
    for (int pc = c0; pc <= c1; ++pc) {
      const int k = pr * S.nc + pc;
      __syncthreads();  // the window loop of the previous term is done with ks and prod (first term: the y patch has landed)
      stage_filter(ks, fb + (long long)k * P.h * P.w, P);
      const float* wk = mult + (long long)k * S.P1 * S.P2;
      const int pi = pr * S.s1 - S.ai, pj = pc * S.s2 - S.aj;  // patch k's origin in y coordinates
      for (int idx = tid; idx < PH * P.PW; idx += 256) {
        const int er = idx / P.PW, ec = idx - er * P.PW;
        const int yi = gi + er + P.off_i, yj = gj + ec + P.off_j;
        const int I = yi - pi, J = yj - pj;
        float v = 0.f;
        if (yi >= 0 && yi < S.Hy && yj >= 0 && yj < S.Wy && I >= 0 && I < S.P1 && J >= 0 && J < S.P2)
          v = (S.xs ? yp[idx] : __ldg(src + (long long)yi * P.Win + yj)) * __ldg(wk + (long long)I * S.P2 + J);
        prod[idx] = v;
      }
      __syncthreads();
      // output rows patch k can reach: [pi, pi + P1 - 1 + h - 1] (y rows [pi, pi + P1) spread by the filter)
      const int ei = pi + S.P1 + P.h - 1, ej = pj + S.P2 + P.w - 1;
      if (wr + 8 <= pi || wr >= ei) continue;  // (warp-uniform)
      float part[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) part[r][q] = 0.f;
      window_fma(prod, ks, P, tx, ty, part);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = oi + ty * 4 + r;
        if (i < pi || i >= ei) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = oj + tx * 4 + q;
          if (j >= pj && j < ej) tot[r][q] += part[r][q];
        }
      }
    }
  }
  store_tile_masked(out + (long long)bc * P.Hout * P.Wout, tot, P, oi, oj, tx, ty);
}

// transpose of replicate / reflect padding: x[p,q] = sum over the extended indices that the padding maps onto (p,q)
// z is the extended image (He = H + h - 1 rows starting at extended index a_min = h/2 - h + 1; same for columns)
__device__ __forceinline__ int preimages(int p, int n, int amin, int amax, int mode, int* start, int* count) {
  // returns the number of ranges; each range is [start, start+count)
  if (mode == 2) {  // replicate
    int lo = p, hi = p;
    if (p == 0) lo = amin;
    if (p == n - 1) hi = amax;
    start[0] = lo; count[0] = hi - lo + 1;
    return 1;
  }
  int k = 0;
  start[k] = p; count[k] = 1; ++k;
  if (p >= 1 && -p >= amin) { start[k] = -p; count[k] = 1; ++k; }
  if (p <= n - 2 && 2 * (n - 1) - p <= amax) { start[k] = 2 * (n - 1) - p; count[k] = 1; ++k; }
  return k;
}

__global__ void __launch_bounds__(256) blur_fold_kernel(const float* __restrict__ z, float* __restrict__ x, int H, int W, int h,
                                                        int w, int mode) {
  const int bc = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W) return;
  const int p = idx / W, q = idx - p * W;
  const int amin = h / 2 - h + 1, amax = H - 1 + h / 2, bmin = w / 2 - w + 1, bmax = W - 1 + w / 2;
  const int We = W + w - 1, He = H + h - 1;
  int rs[3], rc[3], cs[3], cc[3];
  const int nr = preimages(p, H, amin, amax, mode, rs, rc), ncol = preimages(q, W, bmin, bmax, mode, cs, cc);
  const float* zz = z + (long long)bc * He * We;
  float acc = 0.f;
  for (int a = 0; a < nr; ++a)
    for (int ra = rs[a]; ra < rs[a] + rc[a]; ++ra)
      for (int bq = 0; bq < ncol; ++bq)
        for (int cb = cs[bq]; cb < cs[bq] + cc[bq]; ++cb) acc += __ldg(zz + (long long)(ra - amin) * We + (cb - bmin));
  x[(long long)bc * H * W + idx] = acc;
}

static BlurParams corr_params(int C, int Hin, int Win, int Hout, int Wout, int FB, int FC, int h, int w, int flip, int off_i, int off_j,
                              int map, bool align = true) {
  BlurParams P;
  // A tensor-map box has to start on a 16-byte boundary of the image row.  Tiles start at multiples of 64 columns, so the patch
  // origin j0 + off_j is aligned iff off_j is a multiple of 4: prepend shift = off_j mod 4 zero taps to the filter rows and move
  // the origin left by as much (out[j] = sum_v ks'[v] in[j + v + off_j - shift], ks'[v] = ks[v - shift]): same sums, aligned box.
  // align = false keeps the unshifted layout (mapped-loop staging only).
  const int shift = align ? ((off_j % 4) + 4) % 4 : 0;
  off_j -= shift;
  P.shift = shift;
  P.C = C; P.Hin = Hin; P.Win = Win; P.Hout = Hout; P.Wout = Wout; P.h = h; P.w = w; P.wp = (w + shift + 3) & ~3;
  P.FB = FB; P.FC = FC; P.flip = flip; P.off_i = off_i; P.off_j = off_j; P.map = map;
  P.PW = BL_T + P.wp + 4;  // window reads reach column tx*4 + wp + 3
  P.tiles_x = ceil_div(Wout, BL_T);
  return P;
}

constexpr size_t BL_SMEM_BUDGET = 200 * 1024;

static size_t filter_bytes(const BlurParams& P) { return sizeof(float) * (size_t)P.h * P.wp; }
static size_t patch_bytes(const BlurParams& P) { return sizeof(float) * (size_t)(BL_T + P.h - 1) * P.PW; }

// grid + tensor map of one tiled launch over B*C planes of `in` (Hin x Win); use_tma = 0 when the map cannot be built
static int tile_grid(const BlurParams& P, int B, int C, const float* in, bool want_tma, dim3* grid, tt::TileMap* tmap, int* use_tma) {
  const long long tiles = (long long)P.tiles_x * ceil_div(P.Hout, BL_T);
  if ((long long)B * C > 65535 || tiles > 2147483647LL) return set_error(DINVK_EINVAL, "blur: grid too large");
  *grid = dim3((unsigned)tiles, B * C);
  *tmap = tt::TileMap();
  *use_tma = 0;
#ifndef DINVK_EMUL
  if (want_tma && !getenv("DINVK_NO_TMA_STAGING"))
    *use_tma = tt::make_map_f32(tmap, in, P.Win, P.Hin, B * C, P.PW, BL_T + P.h - 1) ? 1 : 0;
#else
  (void)in; (void)want_tma;
#endif
  return DINVK_OK;
}

static int run_corr(const float* in, const float* filt, float* out, int B, int C, int Hin, int Win, int Hout, int Wout,
                    int FB, int FC, int h, int w, int flip, int off_i, int off_j, int map, void* stream) {
  BlurParams P = corr_params(C, Hin, Win, Hout, Wout, FB, FC, h, w, flip, off_i, off_j, map);
  size_t smem = filter_bytes(P) + patch_bytes(P) + 128;
  // The shift taps widen the rows by up to 4 (to the next multiple of 4), and off_j differs between A and A^T: at the budget line
  // the aligned layout of one direction can miss while the other fits.  The unshifted layout, staged by the mapped loop (its box
  // would not be aligned), makes the accepted filters the same in both directions: up to 123 x 123, 1 x 720 and 613 x 1.
  bool aligned = true;
  if (smem > BL_SMEM_BUDGET && P.shift) {
    P = corr_params(C, Hin, Win, Hout, Wout, FB, FC, h, w, flip, off_i, off_j, map, false);
    smem = filter_bytes(P) + patch_bytes(P) + 128;
    aligned = false;
  }
  if (smem > BL_SMEM_BUDGET) return set_error(DINVK_EUNSUPPORTED, "blur: filter %dx%d too large for the tiled kernel", h, w);
  int rc = allow_smem(blur_corr_kernel, smem);
  if (rc) return rc;
  dim3 grid;
  tt::TileMap tmap;
  int use_tma;
  if ((rc = tile_grid(P, B, C, in, aligned, &grid, &tmap, &use_tma))) return rc;
  DINVK_LAUNCH(blur_corr_kernel, grid, dim3(256), smem, stream, tmap, use_tma, in, filt, out, P);
  return DINVK_POST_LAUNCH();
}

// Space-varying forward: the x patch stays in shared memory next to the product patch when both fit the budget Blur uses;
// larger filters (up to Blur's own limit) re-read x for every k instead (L1 / L2 hits: the same tile, K times).
static int run_svblur_fwd(const float* x, const float* mult, const float* filt, float* y, int B, int C, int H, int W, int Hout,
                          int Wout, int MB, int MC, int FB, int FC, int K, int h, int w, int off_i, int off_j, int map, void* stream) {
  SvParams S;
  S.P = corr_params(C, H, W, Hout, Wout, FB, FC, h, w, 1, off_i, off_j, map);
  S.K = K; S.MB = MB; S.MC = MC; S.woff_i = 0; S.woff_j = 0; S.wmap = 0; S.Hm = H; S.Wm = W;
  const size_t one = filter_bytes(S.P) + patch_bytes(S.P) + 128, two = one + patch_bytes(S.P) + 128;
  if (one > BL_SMEM_BUDGET) return set_error(DINVK_EUNSUPPORTED, "svblur: filter %dx%d too large for the tiled kernel", h, w);
  S.xs = two <= BL_SMEM_BUDGET;
  const size_t smem = S.xs ? two : one;
  int rc = allow_smem(svblur_fwd_kernel, smem);
  if (rc) return rc;
  dim3 grid;
  tt::TileMap tmap;
  int use_tma;
  if ((rc = tile_grid(S.P, B, C, x, S.xs, &grid, &tmap, &use_tma))) return rc;
  DINVK_LAUNCH(svblur_fwd_kernel, grid, dim3(256), smem, stream, tmap, use_tma, x, mult, filt, y, S);
  return DINVK_POST_LAUNCH();
}

static int run_svblur_adj(const float* y, const float* mult, const float* filt, float* out, int B, int C, int Hin, int Win, int Hout,
                          int Wout, int MB, int MC, int FB, int FC, int K, int h, int w, int off_i, int off_j, int map, int H, int W,
                          int woff_i, int woff_j, int wmap, void* stream) {
  SvParams S;
  S.P = corr_params(C, Hin, Win, Hout, Wout, FB, FC, h, w, 0, off_i, off_j, map);
  S.K = K; S.MB = MB; S.MC = MC; S.woff_i = woff_i; S.woff_j = woff_j; S.wmap = wmap; S.Hm = H; S.Wm = W; S.xs = 0;
  const size_t smem = filter_bytes(S.P) + patch_bytes(S.P) + 128;
  if (smem > BL_SMEM_BUDGET) return set_error(DINVK_EUNSUPPORTED, "svblur: filter %dx%d too large for the tiled kernel", h, w);
  int rc = allow_smem(svblur_adj_kernel, smem);
  if (rc) return rc;
  dim3 grid;
  tt::TileMap tmap;
  int use_tma;
  if ((rc = tile_grid(S.P, B, C, y, true, &grid, &tmap, &use_tma))) return rc;
  DINVK_LAUNCH(svblur_adj_kernel, grid, dim3(256), smem, stream, tmap, use_tma, y, mult, filt, out, S);
  return DINVK_POST_LAUNCH();
}

// number of patches along one dimension of an n-pixel image padded at the end to the compatible size (utils/_tiling.py:27-46);
// 0 when the image pads to less than one patch
static long long tiled_count(long long n, long long p, long long s) {
  const long long np = (n > p ? n - p : p - n) / s + 1;
  const long long nc = n + (p + np * s - n) % s;
  return nc >= p ? (nc - p) / s + 1 : 0;
}

// fwd: x (H x W) -> y (Ho x Wo), tiles on multiples of 64 of the compatible grid; adj: y -> x (H x W), tiles centred (d = 32).
// The tile grid covers the output plus the d masked rows / columns before it.
static int run_tiled_svblur(bool fwd, const float* in, const float* mult, const float* filt, float* out, int B, int C, int H, int W,
                            int FB, int FC, int K, int nr, int nc, int h, int w, int P1, int P2, int s1, int s2, void* stream) {
  const int Ho = H - h + 1, Wo = W - w + 1;
  TsvParams S;
  S.K = K; S.nr = nr; S.nc = nc; S.P1 = P1; S.P2 = P2; S.s1 = s1; S.s2 = s2;
  S.ai = h / 2; S.aj = w / 2; S.Hy = Ho; S.Wy = Wo;
  S.di = fwd ? S.ai : BL_T / 2; S.dj = fwd ? S.aj : BL_T / 2;
  S.P = fwd ? corr_params(C, H, W, Ho, Wo, FB, FC, h, w, 1, -S.di, -S.dj, 0)
            : corr_params(C, Ho, Wo, H, W, FB, FC, h, w, 0, -(h - 1) - S.di, -(w - 1) - S.dj, 0);
  S.P.tiles_x = ceil_div(S.P.Wout + S.dj, BL_T);
  const size_t one = filter_bytes(S.P) + patch_bytes(S.P) + 128, two = one + patch_bytes(S.P) + 128;
  if (one > BL_SMEM_BUDGET) return set_error(DINVK_EUNSUPPORTED, "tiled_svblur: filter %dx%d too large for the tiled kernel", h, w);
  S.xs = !fwd && two <= BL_SMEM_BUDGET;
  const size_t smem = S.xs ? two : one;
  int rc = fwd ? allow_smem(tiled_svblur_fwd_kernel, smem) : allow_smem(tiled_svblur_adj_kernel, smem);
  if (rc) return rc;
  BlurParams G = S.P;  // the grid: tile_grid counts ceil(Hout / 64) rows of tiles; this grid has d more rows
  G.Hout += S.di;
  dim3 grid;
  tt::TileMap tmap;
  int use_tma;
  if ((rc = tile_grid(G, B, C, in, fwd || S.xs, &grid, &tmap, &use_tma))) return rc;
  if (fwd)
    DINVK_LAUNCH(tiled_svblur_fwd_kernel, grid, dim3(256), smem, stream, tmap, use_tma, in, mult, filt, out, S);
  else
    DINVK_LAUNCH(tiled_svblur_adj_kernel, grid, dim3(256), smem, stream, tmap, use_tma, in, mult, filt, out, S);
  return DINVK_POST_LAUNCH();
}

static int check_blur_args(const void* a, const void* f, const void* o, int B, int C, int H, int W, int FB, int FC, int h, int w,
                           int padding) {
  DINVK_CHECK_ARG(a && f && o, "blur: null pointer");
  DINVK_CHECK_ARG(B >= 0 && C >= 1 && H >= 1 && W >= 1 && h >= 1 && w >= 1, "blur: bad shape");
  DINVK_CHECK_ARG((FB == 1 || FB == B) && (FC == 1 || FC == C), "blur: filter batch/channel (%d,%d) must be 1 or match (%d,%d)", FB, FC, B, C);
  DINVK_CHECK_ARG(padding >= DINVK_PAD_VALID && padding <= DINVK_PAD_CONSTANT, "blur: unknown padding %d", padding);
  DINVK_CHECK_ARG(padding != DINVK_PAD_VALID || (H >= h && W >= w), "blur: valid padding needs an image at least as large as the filter");
  DINVK_CHECK_ARG(padding != DINVK_PAD_REFLECT || (h / 2 < H && w / 2 < W), "blur: reflect padding needs pad < image size");
  return 0;
}

}  // namespace dinvk

using namespace dinvk;

extern "C" int dinvk_blur_fwd(const float* x, const float* filt, float* y, int B, int C, int H, int W, int FB, int FC, int h,
                              int w, int padding, void* stream) {
  int rc = check_blur_args(x, filt, y, B, C, H, W, FB, FC, h, w, padding);
  if (rc) return rc;
  if (B == 0) return DINVK_OK;
  if (padding == DINVK_PAD_VALID) return run_corr(x, filt, y, B, C, H, W, H - h + 1, W - w + 1, FB, FC, h, w, 1, 0, 0, 0, stream);
  const int map = padding == DINVK_PAD_CIRCULAR ? 1 : padding == DINVK_PAD_REPLICATE ? 2 : padding == DINVK_PAD_REFLECT ? 3 : 0;
  return run_corr(x, filt, y, B, C, H, W, H, W, FB, FC, h, w, 1, h / 2 - (h - 1), w / 2 - (w - 1), map, stream);
}

extern "C" size_t dinvk_blur_adj_workspace_bytes(int B, int C, int H, int W, int h, int w, int padding) {
  if (padding == DINVK_PAD_REPLICATE || padding == DINVK_PAD_REFLECT)
    return sizeof(float) * (size_t)B * C * (size_t)(H + h - 1) * (size_t)(W + w - 1) + 256;
  return 256;
}

extern "C" int dinvk_blur_adj(const float* y, const float* filt, float* x, int B, int C, int H, int W, int FB, int FC, int h,
                              int w, int padding, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_blur_args(y, filt, x, B, C, H, W, FB, FC, h, w, padding);
  if (rc) return rc;
  if (B == 0) return DINVK_OK;
  if (padding == DINVK_PAD_VALID)
    return run_corr(y, filt, x, B, C, H - h + 1, W - w + 1, H, W, FB, FC, h, w, 0, -(h - 1), -(w - 1), 0, stream);
  if (padding == DINVK_PAD_CIRCULAR || padding == DINVK_PAD_CONSTANT)
    return run_corr(y, filt, x, B, C, H, W, H, W, FB, FC, h, w, 0, -(h / 2), -(w / 2), padding == DINVK_PAD_CIRCULAR ? 1 : 0, stream);
  // replicate / reflect: zero-extended correlation on the padded domain, then fold the border strips back
  const size_t need = dinvk_blur_adj_workspace_bytes(B, C, H, W, h, w, padding);
  if (!workspace || workspace_bytes < need) return set_error(DINVK_EWORKSPACE, "dinvk_blur_adj: workspace %zu < %zu", workspace_bytes, need);
  float* z = reinterpret_cast<float*>(((uintptr_t)workspace + 127) & ~(uintptr_t)127);
  const int He = H + h - 1, We = W + w - 1;
  // extended output index a' = a - a_min with a_min = h/2 - h + 1: in index = a + u - h/2 = a' + u + (a_min - h/2) = a' + u - (h-1)
  if ((rc = run_corr(y, filt, z, B, C, H, W, He, We, FB, FC, h, w, 0, -(h - 1), -(w - 1), 0, stream))) return rc;
  DINVK_LAUNCH(blur_fold_kernel, dim3(ceil_div((long long)H * W, 256), B * C), dim3(256), 0, stream, (const float*)z, x, H, W, h, w,
               padding == DINVK_PAD_REPLICATE ? 2 : 3);
  return DINVK_POST_LAUNCH();
}

// ---- space-varying blur: deepinv/physics/functional/product_convolution.py:10-68 (product_convolution2d and its adjoint, the
// bodies of SpaceVaryingBlur.A / A_adjoint, deepinv/physics/blur.py:803-849) -------------------------------------------------
static int check_svblur_args(const void* a, const void* m, const void* f, const void* o, int B, int C, int H, int W, int MB, int MC,
                             int FB, int FC, int K, int h, int w, int padding) {
  DINVK_CHECK_ARG(m, "svblur: null multipliers");
  DINVK_CHECK_ARG(K >= 1, "svblur: K = %d terms", K);
  DINVK_CHECK_ARG((MB == 1 || MB == B) && (MC == 1 || MC == C), "svblur: multiplier batch/channel (%d,%d) must be 1 or match (%d,%d)",
                  MB, MC, B, C);
  return check_blur_args(a, f, o, B, C, H, W, FB, FC, h, w, padding);
}

extern "C" int dinvk_svblur_fwd(const float* x, const float* mult, const float* filt, float* y, int B, int C, int H, int W, int MB,
                                int MC, int FB, int FC, int K, int h, int w, int padding, void* stream) {
  int rc = check_svblur_args(x, mult, filt, y, B, C, H, W, MB, MC, FB, FC, K, h, w, padding);
  if (rc) return rc;
  if (B == 0) return DINVK_OK;
  if (padding == DINVK_PAD_VALID)
    return run_svblur_fwd(x, mult, filt, y, B, C, H, W, H - h + 1, W - w + 1, MB, MC, FB, FC, K, h, w, 0, 0, 0, stream);
  const int map = padding == DINVK_PAD_CIRCULAR ? 1 : padding == DINVK_PAD_REPLICATE ? 2 : padding == DINVK_PAD_REFLECT ? 3 : 0;
  return run_svblur_fwd(x, mult, filt, y, B, C, H, W, H, W, MB, MC, FB, FC, K, h, w, h / 2 - (h - 1), w / 2 - (w - 1), map, stream);
}

extern "C" size_t dinvk_svblur_adj_workspace_bytes(int B, int C, int H, int W, int h, int w, int padding) {
  return dinvk_blur_adj_workspace_bytes(B, C, H, W, h, w, padding);
}

extern "C" int dinvk_svblur_adj(const float* y, const float* mult, const float* filt, float* x, int B, int C, int H, int W, int MB,
                                int MC, int FB, int FC, int K, int h, int w, int padding, void* workspace, size_t workspace_bytes,
                                void* stream) {
  int rc = check_svblur_args(y, mult, filt, x, B, C, H, W, MB, MC, FB, FC, K, h, w, padding);
  if (rc) return rc;
  if (B == 0) return DINVK_OK;
  if (padding == DINVK_PAD_VALID)
    return run_svblur_adj(y, mult, filt, x, B, C, H - h + 1, W - w + 1, H, W, MB, MC, FB, FC, K, h, w, -(h - 1), -(w - 1), 0, H, W,
                          0, 0, 0, stream);
  if (padding == DINVK_PAD_CIRCULAR || padding == DINVK_PAD_CONSTANT)
    return run_svblur_adj(y, mult, filt, x, B, C, H, W, H, W, MB, MC, FB, FC, K, h, w, -(h / 2), -(w / 2),
                          padding == DINVK_PAD_CIRCULAR ? 1 : 0, H, W, 0, 0, 0, stream);
  // replicate / reflect: the multiplied sum on the zero-extended domain, then ONE fold (blur_fold_kernel, as dinvk_blur_adj)
  const size_t need = dinvk_svblur_adj_workspace_bytes(B, C, H, W, h, w, padding);
  if (!workspace || workspace_bytes < need) return set_error(DINVK_EWORKSPACE, "dinvk_svblur_adj: workspace %zu < %zu", workspace_bytes, need);
  float* z = reinterpret_cast<float*>(((uintptr_t)workspace + 127) & ~(uintptr_t)127);
  const int He = H + h - 1, We = W + w - 1, mode = padding == DINVK_PAD_REPLICATE ? 2 : 3;
  if ((rc = run_svblur_adj(y, mult, filt, z, B, C, H, W, He, We, MB, MC, FB, FC, K, h, w, -(h - 1), -(w - 1), 0, H, W,
                           h / 2 - h + 1, w / 2 - w + 1, mode, stream)))
    return rc;
  DINVK_LAUNCH(blur_fold_kernel, dim3(ceil_div((long long)H * W, 256), B * C), dim3(256), 0, stream, (const float*)z, x, H, W, h, w, mode);
  return DINVK_POST_LAUNCH();
}

// ---- tiled space-varying blur: deepinv/physics/blur.py:871-1192 (TiledSpaceVaryingBlur.A / A_adjoint) and
// deepinv/physics/functional/tiled_product_convolution.py (the multipliers); valid padding only ------------------------------
static int tiled_svblur(bool fwd, const float* in, const float* mult, const float* filt, float* out, int B, int C, int H, int W,
                        int FB, int FC, int K, int h, int w, int P1, int P2, int s1, int s2, void* stream) {
  DINVK_CHECK_ARG(mult, "tiled_svblur: null multipliers");
  DINVK_CHECK_ARG(P1 >= 1 && P2 >= 1 && s1 >= 1 && s2 >= 1, "tiled_svblur: bad patch (%d,%d) / stride (%d,%d)", P1, P2, s1, s2);
  DINVK_CHECK_ARG(s1 <= P1 && s2 <= P2, "tiled_svblur: stride (%d,%d) larger than the patch (%d,%d)", s1, s2, P1, P2);
  int rc = check_blur_args(in, filt, out, B, C, H, W, FB, FC, h, w, DINVK_PAD_VALID);
  if (rc) return rc;
  const long long nr = tiled_count(H, P1, s1), nc = tiled_count(W, P2, s2);
  DINVK_CHECK_ARG(nr >= 1 && nc >= 1 && nr * nc == K, "tiled_svblur: %lld x %lld patches on a %dx%d image, %d filters", nr, nc, H, W, K);
  if (B == 0) return DINVK_OK;
  return run_tiled_svblur(fwd, in, mult, filt, out, B, C, H, W, FB, FC, K, (int)nr, (int)nc, h, w, P1, P2, s1, s2, stream);
}

extern "C" int dinvk_tiled_svblur_fwd(const float* x, const float* mult, const float* filt, float* y, int B, int C, int H, int W,
                                      int FB, int FC, int K, int h, int w, int P1, int P2, int s1, int s2, void* stream) {
  return tiled_svblur(true, x, mult, filt, y, B, C, H, W, FB, FC, K, h, w, P1, P2, s1, s2, stream);
}

extern "C" int dinvk_tiled_svblur_adj(const float* y, const float* mult, const float* filt, float* x, int B, int C, int H, int W,
                                      int FB, int FC, int K, int h, int w, int P1, int P2, int s1, int s2, void* stream) {
  return tiled_svblur(false, y, mult, filt, x, B, C, H, W, FB, FC, K, h, w, P1, P2, s1, s2, stream);
}
