// radon.cu — parallel-beam Radon transform, its exact transpose, and the IRadon back-projection.
//
// Replaces (reference, relative to the deepinv tree):
//   Radon.forward: pad -> grid_sample over all angles -> sum over rows      physics/functional/radon.py:252-309
//   the autograd adjoint of Tomography.A (exact transpose)                  physics/tomography.py:322-342
//   IRadon.forward(filtering=False): sample the sinogram, sum over angles   physics/functional/radon.py:396-450
//
// The reference materialises a (B,C,P,P*A) rotated stack (378 MB per 512^2 image) and reduces it; here
// every ray / pixel accumulates in a register and the only HBM traffic is the image and the sinogram
// (SURVEY §8d: 50.3 MB per cfg3 call).  These kernels are bound by fp32 issue + L1 gathers, not by HBM.
//
// Geometry: affine_grid/grid_sample(align_corners=True) sample the padded image at
//   lin[k] = linspace(-1,1,P)[k];  g = R_theta (lin[j], lin[i]);  pix = ((g + 1) / 2) * (P - 1)
// i.e., in exact arithmetic, pix_x = cx + c (j - cx) + s (i - cx), pix_y = cx - s (j - cx) + c (i - cx), cx = (P-1)/2.  The
// reference evaluates the first form in fp32: a coordinate of magnitude ~P/2 then carries ~P * 3e-8 of rounding, which is
// what its results are off by at 512 x 512 (2e-5 .. 4e-5 relative, tests/test_gpu_radon_tiled.py).  The Radon kernels
// evaluate the second form in fp64 (cos / sin arrive as fp32 (hi, lo) pairs, one DADD per coordinate and step along a
// sample), so they sit closer to the exact operator than the reference itself; bilinear weights from floor(pix) as fp32,
// zeros outside.  Sinograms are stored ANGLE-major (BC, A, P): this is
//   the memory the reference returns as the transposed view (B,C,P,A) (radon.py:291-293).
#include "common.cuh"
#include "tma_tile.cuh"
#ifndef DINVK_EMUL
#include <cstdlib>
#endif

namespace dinvk {

struct RadonGeom {
  int W, P, A, pb, circle;
  float step;  // linspace step 2/(P-1) in fp32
};

// torch.linspace(-1, 1, P) in fp32 (symmetric evaluation, ATen RangeFactories)
__device__ __forceinline__ float lin_at(int k, int P, float step) {
  return (k < P / 2) ? (-1.0f + step * (float)k) : (1.0f - step * (float)(P - 1 - k));
}

// Sample coordinates in 64-bit FIXED POINT with 45 fractional bits (Q45): with U = 2j - (P-1), V = 2i - (P-1) (integers)
//   PX(i, j) = cx Q45 + (C45 U + S45 V) / 2,   PY(i, j) = cx Q45 + (C45 V - S45 U) / 2,   C45 = round(cos 2^45), S45 likewise
// Integer arithmetic is exact and associative: stepping along a ray is PX += S45, PY += C45 and gives bit for bit the value of
// the closed form, so every tile / kernel family sees the same position for a sample (the owner tile of a sample is decided
// by floor(px), floor(py)).  cos/sin carry 2^-46 of rounding -> positions are good to ~1e-11 pixels.
struct Trig45 { long long c, s; };
__device__ __forceinline__ Trig45 trig45(const float* __restrict__ cos_t, const float* __restrict__ sin_t, int A, int t) {
  // tables: A fp32 values followed by their A low-order parts (value = hi + lo)
  const double sc = 35184372088832.0;  // 2^45
  Trig45 r;
  r.c = __double2ll_rn(((double)__ldg(cos_t + t) + (double)__ldg(cos_t + A + t)) * sc);
  r.s = __double2ll_rn(((double)__ldg(sin_t + t) + (double)__ldg(sin_t + A + t)) * sc);
  return r;
}
__device__ __forceinline__ void sample_pos45(const Trig45& T, int P, int j, int i, long long& PX, long long& PY) {
  const long long U = 2LL * j - (P - 1), V = 2LL * i - (P - 1), CX = (long long)(P - 1) << 44;  // (P-1)/2 in Q45
  PX = CX + ((T.c * U + T.s * V) >> 1);
  PY = CX + ((T.c * V - T.s * U) >> 1);
}
// integer cell and the two fp32 bilinear weights of one coordinate
__device__ __forceinline__ void cell_weights(long long Q, int& cell, float& w0, float& w1) {
  cell = (int)(Q >> 45);
  w1 = (float)(unsigned)((unsigned long long)Q >> 13) * 2.3283064365386963e-10f;  // top 32 fractional bits * 2^-32
  w0 = 1.0f - w1;
}

__device__ __forceinline__ void sample_pos(float c, float s, float xj, float yi, float pm1, float& px, float& py) {
  const float gx = fmaf(s, yi, c * xj);
  const float gy = fmaf(c, yi, -s * xj);
  px = ((gx + 1.0f) * 0.5f) * pm1;
  py = ((gy + 1.0f) * 0.5f) * pm1;
}

// image value at padded coordinates (X,Y): zero padding outside the W x W support; optional inscribed disc
__device__ __forceinline__ float img_at(const float* __restrict__ img, const RadonGeom& G, int X, int Y) {
  const int x = X - G.pb, y = Y - G.pb;
  if (x < 0 || x >= G.W || y < 0 || y >= G.W) return 0.f;
  float v = __ldg(img + (long long)y * G.W + x);
  if (G.circle) {
    const float ax = 2.0f * (float)x / (float)(G.W - 1) - 1.0f, ay = 2.0f * (float)y / (float)(G.W - 1) - 1.0f;
    if (!(ax * ax + ay * ay <= 1.0f)) v = 0.f;
  }
  return v;
}

// one thread per ray (bc, t, j): sino[bc, t, j] = scale * sum_i bilinear(x_pad, S_t(i, j))
__global__ void __launch_bounds__(128) radon_fwd_kernel(const float* __restrict__ x, float* __restrict__ sino, RadonGeom G,
                                                        const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                        float scale) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y, bc = blockIdx.z;
  if (j >= G.P) return;
  const float c = __ldg(cos_t + t), s = __ldg(sin_t + t);
  const float pm1 = (float)(G.P - 1);
  const float* img = x + (long long)bc * G.W * G.W;
  // conservative row range in which the sample can touch the image support [pb-1, pb+W] (both axes):
  // pix_x ~ cx + c (j-cx) + s (i-cx),  pix_y ~ cx - s (j-cx) + c (i-cx)
  const float cx = 0.5f * pm1;
  const float lo = (float)G.pb - 1.0f, hi = (float)(G.pb + G.W);
  float i_lo = 0.f, i_hi = pm1;
  {
    const float bx = cx + c * ((float)j - cx), by = cx - s * ((float)j - cx);
    // lo < bx + s*(i-cx) < hi   and   lo < by + c*(i-cx) < hi
    if (fabsf(s) > 1e-6f) {
      float a = (lo - bx) / s + cx, b = (hi - bx) / s + cx;
      if (a > b) { const float tmp = a; a = b; b = tmp; }
      i_lo = fmaxf(i_lo, a); i_hi = fminf(i_hi, b);
    } else if (!(bx > lo - 1.f && bx < hi + 1.f)) { i_hi = -1.f; }
    if (fabsf(c) > 1e-6f) {
      float a = (lo - by) / c + cx, b = (hi - by) / c + cx;
      if (a > b) { const float tmp = a; a = b; b = tmp; }
      i_lo = fmaxf(i_lo, a); i_hi = fminf(i_hi, b);
    } else if (!(by > lo - 1.f && by < hi + 1.f)) { i_hi = -1.f; }
  }
  const int i0 = max(0, (int)floorf(i_lo) - 2), i1 = min(G.P - 1, (int)ceilf(i_hi) + 2);
  float acc = 0.f;
  const Trig45 tq = trig45(cos_t, sin_t, G.A, t);
  long long PX, PY;
  // (a ray that misses the support has i0 > i1 and possibly i0 far beyond P: its start position is never used, but is kept in
  // range so the Q45 products cannot overflow)
  sample_pos45(tq, G.P, j, min(i0, G.P - 1), PX, PY);
  for (int i = i0; i <= i1; ++i, PX += tq.s, PY += tq.c) {
    int X0, Y0;
    float wx0, wx1, wy0, wy1;
    cell_weights(PX, X0, wx0, wx1);
    cell_weights(PY, Y0, wy0, wy1);
    if (X0 < G.pb - 1 || X0 >= G.pb + G.W || Y0 < G.pb - 1 || Y0 >= G.pb + G.W) continue;
    const float v00 = img_at(img, G, X0, Y0), v01 = img_at(img, G, X0 + 1, Y0);
    const float v10 = img_at(img, G, X0, Y0 + 1), v11 = img_at(img, G, X0 + 1, Y0 + 1);
    acc += v00 * (wx0 * wy0) + v01 * (wx1 * wy0) + v10 * (wx0 * wy1) + v11 * (wx1 * wy1);
  }
  sino[((long long)bc * G.A + t) * G.P + j] = acc * scale;
}

// exact transpose, gather form: one thread per image pixel.  For each angle the sample lattice is the
// unit grid rotated about the centre; the samples whose bilinear footprint covers pixel (X,Y) lie within
// sqrt(2) of its lattice coordinates, i.e. among the 3x3 lattice points around the nearest one.
__global__ void __launch_bounds__(256) radon_adj_kernel(const float* __restrict__ sino, float* __restrict__ x, RadonGeom G,
                                                        const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                        float scale) {
  DINVK_DYN_SMEM(long long, s_cs);  // cos[A], sin[A] in Q45
  for (int k = threadIdx.x; k < G.A; k += blockDim.x) { const Trig45 q = trig45(cos_t, sin_t, G.A, k); s_cs[k] = q.c; s_cs[G.A + k] = q.s; }
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int bc = blockIdx.y;
  const bool active = p < G.W * G.W;
  const int yy = active ? p / G.W : 0, xx = active ? p - yy * G.W : 0;
  const int X = xx + G.pb, Y = yy + G.pb;
  const float pm1 = (float)(G.P - 1), cx = 0.5f * pm1;
  const float dx = (float)X - cx, dy = (float)Y - cx;
  const float* sbase = sino + (long long)bc * G.A * G.P;
  float acc = 0.f;
  if (active) {
    for (int t = 0; t < G.A; ++t) {
      Trig45 tq;
      tq.c = s_cs[t]; tq.s = s_cs[G.A + t];
      const float c = (float)tq.c * 2.842170943040401e-14f, s = (float)tq.s * 2.842170943040401e-14f;  // * 2^-45
      const int jc = __float2int_rn(cx + c * dx - s * dy), ic = __float2int_rn(cx + s * dx + c * dy);
      const float* srow = sbase + (long long)t * G.P;
#pragma unroll
      for (int dj = -1; dj <= 1; ++dj) {
        const int j = jc + dj;
        if (j < 0 || j >= G.P) continue;
        float wsum = 0.f;
#pragma unroll
        for (int di = -1; di <= 1; ++di) {
          const int i = ic + di;
          if (i < 0 || i >= G.P) continue;
          long long PX, PY;
          sample_pos45(tq, G.P, j, i, PX, PY);
          int X0, Y0;
          float wx0, wx1, wy0, wy1;
          cell_weights(PX, X0, wx0, wx1);
          cell_weights(PY, Y0, wy0, wy1);
          const float wx = (X0 == X) ? wx0 : ((X0 + 1 == X) ? wx1 : 0.f);
          const float wy = (Y0 == Y) ? wy0 : ((Y0 + 1 == Y) ? wy1 : 0.f);
          wsum += wx * wy;
        }
        acc = fmaf(__ldg(srow + j), wsum, acc);
      }
    }
    if (G.circle) {
      const float ax = 2.0f * (float)xx / (float)(G.W - 1) - 1.0f, ay = 2.0f * (float)yy / (float)(G.W - 1) - 1.0f;
      if (!(ax * ax + ay * ay <= 1.0f)) acc = 0.f;
    }
    x[(long long)bc * G.W * G.W + p] = acc * scale;
  }
}

// IRadon back-projection: reco[y,x] = scale * sum_t bilinear(sino as a (P x A) image, col = f(t), row = T(x,y,t))
__global__ void __launch_bounds__(256) iradon_bp_kernel(const float* __restrict__ sino, float* __restrict__ x, RadonGeom G,
                                                        const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                        float scale) {
  DINVK_DYN_SMEM(float, s_cs);
  for (int k = threadIdx.x; k < G.A; k += blockDim.x) { s_cs[k] = __ldg(cos_t + k); s_cs[G.A + k] = __ldg(sin_t + k); }
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int bc = blockIdx.y;
  if (p >= G.W * G.W) return;
  const int yy = p / G.W, xx = p - yy * G.W;
  const float xg = lin_at(xx + G.pb, G.P, G.step), yg = lin_at(yy + G.pb, G.P, G.step);
  const float pm1 = (float)(G.P - 1), am1 = (float)(G.A - 1);
  const float* sbase = sino + (long long)bc * G.A * G.P;
  float acc = 0.f;
  for (int t = 0; t < G.A; ++t) {
    const float T = xg * s_cs[t] - yg * s_cs[G.A + t];
    const float Xn = ((1.0f * (float)t) * 2.0f) / am1 - 1.0f;
    const float pxs = ((Xn + 1.0f) * 0.5f) * am1;  // column (angle) coordinate
    const float pys = ((T + 1.0f) * 0.5f) * pm1;   // row (detector) coordinate
    const float fx = floorf(pxs), fy = floorf(pys);
    const int c0 = (int)fx, r0 = (int)fy;
    const float wx1 = pxs - fx, wy1 = pys - fy, wx0 = (fx + 1.0f) - pxs, wy0 = (fy + 1.0f) - pys;
    float v = 0.f;
#pragma unroll
    for (int dc = 0; dc < 2; ++dc) {
      const int cc = c0 + dc;
      if (cc < 0 || cc >= G.A) continue;
      const float wx = dc ? wx1 : wx0;
      if (wx == 0.f) continue;
      const float* col = sbase + (long long)cc * G.P;  // angle-major storage: column cc of the (P x A) image is contiguous
      if (r0 >= 0 && r0 < G.P) v += __ldg(col + r0) * (wx * wy0);
      if (r0 + 1 >= 0 && r0 + 1 < G.P) v += __ldg(col + r0 + 1) * (wx * wy1);
    }
    acc += v;
  }
  if (G.circle && !(xg * xg + yg * yg <= 1.0f)) acc = 0.f;
  x[(long long)bc * G.W * G.W + p] = acc * scale;
}


// ---------------------------------------------------------------------------------------------------------------------
// Tiled forward projection and exact transpose (the default path on the GPU).
//
// A CTA owns one 64 x 64-pixel tile of one image for ALL angles: the tile (+1 pixel halo, 66 x 68) is staged once in
// shared memory with explicit zeros outside the image — the reference's zero padding (radon.py:262-266), so the sqrt(2)
// padded image never exists — and every bilinear tap of the 47 M samples per image that fall in the image support is a
// shared-memory access instead of an L1 gather (the ray-per-thread kernel above is bound by L1 tag lookups: a warp of
// adjacent rays touches up to 32 cache lines per tap).  Each sample (i, j) of the rotated lattice is owned by exactly
// one tile (the one that contains floor(px), floor(py)); a warp takes one angle at a time, its lanes adjacent rays,
// each lane walks the clipped range of steps i of its ray and accumulates in a register.
//   forward:   lane partial sums -> one fp32 atomicAdd per (tile, angle, ray) into the zeroed sinogram
//   transpose: lane reads sino[t, j] once, scatters w * y into the zeroed shared tile (shared-memory atomics, same
//              fp32 weights as the forward => <Ax, y> = <x, A^T y> up to summation order), tile added to the image at the end
// Sample geometry is evaluated with the same fp32 formulas as above.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int RT = 64;    // tile edge (pixels)
constexpr int RTW = 76;   // staged row pitch / box width (floats): columns ox-3 .. ox+72 (76 % 32 = 12: rows 12 banks apart, like the 4 of the first 68-float pitch; 72 costs 8 % in bank conflicts) — a tensor-map box must start on a 16-byte
                          // boundary of the image row, and ox - 3 = 64 tx - 4 is a multiple of 4 (the first attempts, round 1 and
                          // this round, started the box at ox = 64 tx - 1 and trapped as an illegal instruction)
constexpr int RXO = 3;    // index of column ox inside a staged row
constexpr int RTH = 66;   // staged rows
// transpose: columns 69 .. 75 of each accumulator row are never added to (the owned floors end at offset 64, their right taps at
// 65 = column 68); columns RNF .. RNF+4 hold 2 bits per owned floor cell of the row (65 cells) that mark NaN / Inf samples
constexpr int RNF = 70;
constexpr int RT_THREADS = 128;

// steps i of ray j whose sample can fall in the tile [fxl, fxu) x [fyl, fyu) (padded coordinates), +- 2 steps of margin for the
// fp32 estimate: fxl <= bx + s (i - cx) < fxu and fyl <= by + c (i - cx) < fyu
__device__ __forceinline__ void tile_steps(float c, float s, int j, float cx, float pm1, int P, float fxl, float fxu, float fyl,
                                           float fyu, int& i0, int& i1) {
  float i_lo = 0.f, i_hi = pm1;
  const float bx = cx + c * ((float)j - cx), by = cx - s * ((float)j - cx);
  if (fabsf(s) > 1e-6f) {
    float a = (fxl - bx) / s + cx, b = (fxu - bx) / s + cx;
    if (a > b) { const float tmp = a; a = b; b = tmp; }
    i_lo = fmaxf(i_lo, a); i_hi = fminf(i_hi, b);
  } else if (!(bx > fxl - 1.f && bx < fxu + 1.f)) { i_hi = -1.f; }
  if (fabsf(c) > 1e-6f) {
    float a = (fyl - by) / c + cx, b = (fyu - by) / c + cx;
    if (a > b) { const float tmp = a; a = b; b = tmp; }
    i_lo = fmaxf(i_lo, a); i_hi = fminf(i_hi, b);
  } else if (!(by > fyl - 1.f && by < fyu + 1.f)) { i_hi = -1.f; }
  i0 = max(0, (int)floorf(i_lo) - 2);
  i1 = min(P - 1, (int)ceilf(i_hi) + 2);
}

// rays j of angle (c, s) that can reach the tile [fxl, fxu) x [fyl, fyu): j ~ cx + c (X - cx) - s (Y - cx) over its corners, +- 1
__device__ __forceinline__ void tile_rays(float c, float s, float cx, int P, float fxl, float fxu, float fyl, float fyu, int& jmin,
                                          int& jmax) {
  const float j00 = c * (fxl - cx) - s * (fyl - cx), j10 = c * (fxu - cx) - s * (fyl - cx);
  const float j01 = c * (fxl - cx) - s * (fyu - cx), j11 = c * (fxu - cx) - s * (fyu - cx);
  jmin = max(0, (int)floorf(cx + fminf(fminf(j00, j10), fminf(j01, j11))) - 1);
  jmax = min(P - 1, (int)ceilf(cx + fmaxf(fmaxf(j00, j10), fmaxf(j01, j11))) + 1);
}

// non-finite samples of the transpose, by floor cell (ux, uy) of the tile: 1 = +Inf, 2 = -Inf, 3 = NaN, ORed (+Inf and -Inf
// together give NaN, as in an fp32 sum)
__device__ __forceinline__ void mark_nonfinite(int* TI, int ux, int uy, float v) {
  const int code = (v != v) ? 3 : (v > 0.f ? 1 : 2);
  atomicOr(TI + uy * RTW + RNF + (ux >> 4), code << (2 * (ux & 15)));
}
__device__ __forceinline__ int nonfinite_mark(const int* TI, int ux, int uy) {
  if (ux < 0 || uy < 0 || ux > RT || uy > RT) return 0;
  return (TI[uy * RTW + RNF + (ux >> 4)] >> (2 * (ux & 15))) & 3;
}

template <bool ADJ>
__global__ void __launch_bounds__(RT_THREADS) radon_tiled_kernel(const __grid_constant__ tt::TileMap tmap, int use_tma,
                                                                 const float* __restrict__ src,
                                                                 float* __restrict__ out, RadonGeom G, const float* __restrict__ cos_t,
                                                                 const float* __restrict__ sin_t, float scale, int tps) {
#ifdef DINVK_EMUL
  unsigned char* rt_raw = reinterpret_cast<unsigned char*>(::emul::dyn_smem());
#else
  extern __shared__ __align__(128) unsigned char rt_raw[];
#endif
  // forward: the staged image tile, fp32 [RTH][RTW].  transpose: the tile's accumulator in 32-bit FIXED POINT [RTH][RTW] (scale per tile, see below): an fp32
  // (or 64-bit) atomicAdd on shared memory is a compare-and-swap loop (SASS ATOMS.CAST.SPIN: the first version's transpose took
  // 2x the forward), a 32-bit integer add without return value is ONE fire-and-forget ATOMS.ADD, and integer sums do not
  // depend on the order of the adds (the tile's result is deterministic)
  // (the tile is the destination of a tensor-map copy: 128-byte aligned at run time — the declared alignment of a dynamic
  // shared array is not honoured beyond 16 bytes when the kernel also has static shared variables; the launch reserves the slack)
  unsigned char* rt_al = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(rt_raw) + 127) & ~static_cast<uintptr_t>(127));
  float* T = reinterpret_cast<float*>(rt_al);
  int* TI = reinterpret_cast<int*>(rt_al);
  long long* s_cs = reinterpret_cast<long long*>(rt_al + (((size_t)RTH * RTW * 4 + 15) & ~(size_t)15));  // cos[A], sin[A], Q45
  __shared__ unsigned s_absmax[2];  // transpose: max |y| over the tile's rays, max over the finite ones
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ty = blockIdx.x / tps, tx = blockIdx.x - ty * tps;
  const int bc = blockIdx.y;
  // tile origin in image coordinates (first staged pixel) and in padded coordinates
  const int ox = RT * tx - 1, oy = RT * ty - 1;
  const int xl = G.pb + ox, yl = G.pb + oy;
  // owned floor coordinates: offsets 0 .. xr (the last tile also owns the floor W-1, whose right tap is the zero padding)
  const int xr = (tx == tps - 1) ? (G.W - 1 - ox) : (RT - 1);
  const int yr = (ty == tps - 1) ? (G.W - 1 - oy) : (RT - 1);

  if (!ADJ) {
    // stage the tile once; zeros outside the image = the reference's zero padding (radon.py:262-266)
#ifndef DINVK_EMUL
    if (use_tma) {
      // ONE tensor-map box load (68 x 66 fp32, origin (ox, oy) may be -1): the copy engine zero-fills what lies outside the image
      __shared__ __align__(8) uint64_t tile_bar;
      tt::stage_tile(T, &tmap, &tile_bar, ox - RXO, oy, bc, RTH * RTW * 4);
    } else
#endif
    {
      const float* img = src + (long long)bc * G.W * G.W;
      for (int e = tid; e < RTH * RTW; e += RT_THREADS) {
        const int uy = e / RTW, ux = e - uy * RTW;
        const int x = ox - RXO + ux, y = oy + uy;
        T[e] = (x >= 0 && x < G.W && y >= 0 && y < G.W) ? __ldg(img + (long long)y * G.W + x) : 0.f;
      }
    }
  } else {
    for (int e = tid; e < RTH * RTW; e += RT_THREADS) TI[e] = 0;
    if (tid == 0) { s_absmax[0] = 0u; s_absmax[1] = 0u; }
  }
  for (int k = tid; k < G.A; k += RT_THREADS) { const Trig45 q = trig45(cos_t, sin_t, G.A, k); s_cs[k] = q.c; s_cs[G.A + k] = q.s; }
  __syncthreads();
  if (!ADJ) {
    if (G.circle) {  // inscribed-disc mask of the image (radon.py:268-279), applied once to the staged tile
      for (int e = tid; e < RTH * RTW; e += RT_THREADS) {
        const int uy = e / RTW, ux = e - uy * RTW;
        const int x = ox - RXO + ux, y = oy + uy;
        const float ax = 2.0f * (float)x / (float)(G.W - 1) - 1.0f, ay = 2.0f * (float)y / (float)(G.W - 1) - 1.0f;
        if (!(ax * ax + ay * ay <= 1.0f)) T[e] = 0.f;
      }
      __syncthreads();
    }
  }

  const float pm1 = (float)(G.P - 1), cx = 0.5f * pm1;
  const float fxl = (float)xl, fxu = (float)(xl + xr + 1), fyl = (float)yl, fyu = (float)(yl + yr + 1);
  const long long srow0 = (long long)bc * G.A * G.P;
  float fx_scale = 1.f;
  double fx_inv = 1.0;
  if (ADJ) {
    // fixed-point scale of this tile: sf = 0.999 * 2^30 / (2 A m), m = max |y| over the finite values of the rays that can
    // reach the tile (the bits of a non-negative float order like unsigned integers; NaN and Inf order above every finite
    // value and are left out: the pixels they reach are marked and overwritten, see below).  At one angle the bilinear weights of the lattice
    // samples around a pixel sum to between 0.83 and 1 + 4 (1 - 1/sqrt(2))^2 = 1.343 (a tent function summed over a rotated
    // unit lattice; the maximum is at 45 degrees on a lattice point, tests/test_radon_ref64.py), bounded here by 2: a pixel
    // collects at most 1.343 A m < 2 A m, i.e. < 2^30 after scaling — no overflow.  One unit is 2 A m / 2^30 (A = 180:
    // 3.4e-7 m); the rounding errors of a pixel's ~4 A contributions add up like a random walk to ~8 units: 2.6e-6 m, i.e.
    // 1e-6 .. 2e-6 of the pixel value for white-noise and for ramp-filtered sinograms — an order of magnitude below the fp32
    // coordinate noise of the reference's own transpose at this size, and independent of the order of the adds.
    // (NaN and Inf order above every finite value: when the first sweep meets one, a second takes the largest finite |y|)
    for (int pass = 0; pass < 2; ++pass) {
      unsigned m = 0u;
      for (int t = warp; t < G.A; t += RT_THREADS / 32) {
        const float c = (float)s_cs[t] * 2.842170943040401e-14f, s = (float)s_cs[G.A + t] * 2.842170943040401e-14f;
        int jmin, jmax;
        tile_rays(c, s, cx, G.P, fxl, fxu, fyl, fyu, jmin, jmax);
        for (int j = jmin + lane; j <= jmax; j += 32) {
          const unsigned b = __float_as_uint(fabsf(__ldg(src + srow0 + (long long)t * G.P + j) * scale));
          m = max(m, (pass == 0 || b < 0x7f800000u) ? b : 0u);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) atomicMax(&s_absmax[pass], m);
      __syncthreads();
      if (s_absmax[0] < 0x7f800000u) break;
    }
    const float mf = __uint_as_float(s_absmax[s_absmax[0] < 0x7f800000u ? 0 : 1]);
    if (mf > 0.f) {
      fx_scale = (0.999f * 1073741824.0f / (float)(2 * G.A)) / mf;
      if (!(fx_scale < 3.0e38f)) fx_scale = 3.0e38f;   // denormal-sized sinograms
    }
    fx_inv = 1.0 / (double)fx_scale;
  }
  if (ADJ && s_absmax[0] >= 0x7f800000u) {
    // a NaN / Inf ray cannot go through the integer accumulator (NaN would convert to 0, Inf saturate and wrap): this pass
    // marks the floor cells of its samples in the tile (RNF); the final add turns the four taps of a marked cell into that
    // non-finite value, whatever the main loop's integer adds left there.  Marks only, in shared memory, and before the main loop: so placed, the kernel keeps the 48 registers
    // it has without this pass (fp32 atomics to the image from a pass after the main loop took 60).
    for (int t = warp; t < G.A; t += RT_THREADS / 32) {
      Trig45 tq;
      tq.c = s_cs[t]; tq.s = s_cs[G.A + t];
      const float c = (float)tq.c * 2.842170943040401e-14f, s = (float)tq.s * 2.842170943040401e-14f;
      int jmin, jmax;
      tile_rays(c, s, cx, G.P, fxl, fxu, fyl, fyu, jmin, jmax);
      for (int j = jmin + lane; j <= jmax; j += 32) {
        const float yv = __ldg(src + srow0 + (long long)t * G.P + j) * scale;
        if (fabsf(yv) <= 3.402823466e38f) continue;
        int i0, i1;
        tile_steps(c, s, j, cx, pm1, G.P, fxl, fxu, fyl, fyu, i0, i1);
        long long PX, PY;
        sample_pos45(tq, G.P, j, min(i0, G.P - 1), PX, PY);
        for (int i = i0; i <= i1; ++i, PX += tq.s, PY += tq.c) {
          const unsigned ux = (unsigned)((int)(PX >> 45) - xl), uy = (unsigned)((int)(PY >> 45) - yl);
          if (ux > (unsigned)xr || uy > (unsigned)yr) continue;
          mark_nonfinite(TI, ux, uy, yv);
        }
      }
    }
  }
  for (int t = warp; t < G.A; t += RT_THREADS / 32) {
    Trig45 tq;
    tq.c = s_cs[t]; tq.s = s_cs[G.A + t];
    const float c = (float)tq.c * 2.842170943040401e-14f, s = (float)tq.s * 2.842170943040401e-14f;
    int jmin, jmax;
    tile_rays(c, s, cx, G.P, fxl, fxu, fyl, fyu, jmin, jmax);
    for (int j = jmin + lane; j <= jmax; j += 32) {
      int i0, i1;
      tile_steps(c, s, j, cx, pm1, G.P, fxl, fxu, fyl, fyu, i0, i1);
      float acc = 0.f;
      float yv = 0.f;
      if (ADJ && i0 <= i1) yv = (__ldg(src + srow0 + (long long)t * G.P + j) * scale) * fx_scale;
      // (a NaN / Inf ray's integer adds land only on the taps of the cells the pass above marked, which the final add overwrites)
      bool any = false;
      long long PX, PY;
      sample_pos45(tq, G.P, j, min(i0, G.P - 1), PX, PY);  // i0 > i1 (not used) may lie far beyond P, see radon_fwd_kernel
      for (int i = i0; i <= i1; ++i, PX += tq.s, PY += tq.c) {
        int X0, Y0;
        float wx0, wx1, wy0, wy1;
        cell_weights(PX, X0, wx0, wx1);
        cell_weights(PY, Y0, wy0, wy1);
        const unsigned ux = (unsigned)(X0 - xl), uy = (unsigned)(Y0 - yl);
        if (ux > (unsigned)xr || uy > (unsigned)yr) continue;
        if (!ADJ) {
          const float* tp = T + uy * RTW + ux + RXO;
          acc += tp[0] * (wx0 * wy0) + tp[1] * (wx1 * wy0) + tp[RTW] * (wx0 * wy1) + tp[RTW + 1] * (wx1 * wy1);
          any = true;
        } else {
          int* tp = TI + uy * RTW + ux + RXO;
          atomicAdd(tp, __float2int_rn(yv * (wx0 * wy0)));
          atomicAdd(tp + 1, __float2int_rn(yv * (wx1 * wy0)));
          atomicAdd(tp + RTW, __float2int_rn(yv * (wx0 * wy1)));
          atomicAdd(tp + RTW + 1, __float2int_rn(yv * (wx1 * wy1)));
        }
      }
      if (!ADJ && any) atomicAdd(out + srow0 + (long long)t * G.P + j, acc * scale);
    }
  }
  if (ADJ) {
    __syncthreads();
    float* img = out + (long long)bc * G.W * G.W;
    for (int e = tid; e < RTH * RTH; e += RT_THREADS) {
      const int uy = e / RTH, ux = e - uy * RTH;
      const int x = ox + ux, y = oy + uy;
      if (x < 0 || x >= G.W || y < 0 || y >= G.W) continue;
      float v = (float)((double)TI[uy * RTW + ux + RXO] * fx_inv);
      if (s_absmax[0] >= 0x7f800000u) {  // the taps (ux, uy) of the cells (ux - 1 .. ux, uy - 1 .. uy)
        const int code = nonfinite_mark(TI, ux, uy) | nonfinite_mark(TI, ux - 1, uy) | nonfinite_mark(TI, ux, uy - 1) |
                         nonfinite_mark(TI, ux - 1, uy - 1);
        if (code) v = __uint_as_float(code == 1 ? 0x7f800000u : (code == 2 ? 0xff800000u : 0x7fc00000u));
      }
      if (G.circle) {
        const float ax = 2.0f * (float)x / (float)(G.W - 1) - 1.0f, ay = 2.0f * (float)y / (float)(G.W - 1) - 1.0f;
        if (!(ax * ax + ay * ay <= 1.0f)) v = 0.f;
      }
      if (v != 0.f) atomicAdd(img + (long long)y * G.W + x, v);
    }
  }
}

static bool tiled_ok(const void* img, int W, int A) {
  if (getenv("DINVK_NO_TILED_RADON")) return false;
  return W >= RT && (W % 4) == 0 && A <= 2048 && (reinterpret_cast<uintptr_t>(img) & 15) == 0;
}
// returns -1 when the tiled path does not apply
static int launch_tiled(bool adj, const float* x_img, const float* sino_in, float* out, int BC, const RadonGeom& G, const float* cos_t,
                        const float* sin_t, float scale, void* stream) {
  const int tps = (G.W + RT - 1) / RT;
  const size_t smem = (size_t)RTH * RTW * 4 + 16 + (size_t)(2 * G.A + 2) * 8 + 128;
  const size_t out_bytes = adj ? (size_t)BC * G.W * G.W * 4 : (size_t)BC * G.A * G.P * 4;
  if (cudaMemsetAsync(out, 0, out_bytes, (cudaStream_t)stream) != cudaSuccess) return set_error(DINVK_ECUDA, "radon: memset failed");
  int rc;
  tt::TileMap tmap = tt::TileMap();
  int use_tma = 0;
#ifndef DINVK_EMUL
  if (!adj && !getenv("DINVK_NO_TMA_STAGING")) use_tma = tt::make_map_f32(&tmap, x_img, G.W, G.W, BC, RTW, RTH) ? 1 : 0;
#endif
  if (adj) {
    if ((rc = allow_smem(radon_tiled_kernel<true>, smem))) return rc;
    DINVK_LAUNCH(radon_tiled_kernel<true>, dim3(tps * tps, BC), dim3(RT_THREADS), smem, stream, tmap, use_tma, sino_in, out, G, cos_t, sin_t, scale, tps);
  } else {
    if ((rc = allow_smem(radon_tiled_kernel<false>, smem))) return rc;
    DINVK_LAUNCH(radon_tiled_kernel<false>, dim3(tps * tps, BC), dim3(RT_THREADS), smem, stream, tmap, use_tma, x_img, out, G, cos_t, sin_t, scale, tps);
  }
  return DINVK_POST_LAUNCH();
}


// ---- fan-beam projector and its exact transpose (physics/functional/radon.py:16-52 + 252-309 with fan_beam=True) ----
// The reference samples the padded image on a grid that is, for angle t, the rotation of the points
//   (x_i, y_j * d_i),  x_i = linspace(-1,1,G)[i],  y_j = linspace(-1,1,D)[j],  d_i = (half_len * (x_i + src)) / den
// (a fan of straight rays: the detector coordinate scales linearly with the distance from the source) and sums over i.
// One thread per ray (bc, t, j) walks its G samples; the forward gathers into a register, the transpose scatters
// y[t,j] * w with the forward's fp32 weights (global fp32 atomics into the zeroed image).
struct FanGeom {
  int W, G, D, A, pb, circle;
  float step_g, step_d, half_len, src, den;
};

template <bool ADJ>
__global__ void __launch_bounds__(128) fanbeam_kernel(const float* __restrict__ src, float* __restrict__ dst, FanGeom F,
                                                      const float* __restrict__ cos_t, const float* __restrict__ sin_t,
                                                      float scale) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y, bc = blockIdx.z;
  if (j >= F.D) return;
  const float c = __ldg(cos_t + t), s = __ldg(sin_t + t);
  const float gm1 = (float)(F.G - 1);
  const float yj = lin_at(j, F.D, F.step_d);
  RadonGeom R;
  R.W = F.W; R.P = F.G; R.A = F.A; R.pb = F.pb; R.circle = F.circle; R.step = F.step_g;
  const long long WW = (long long)F.W * F.W;
  const float* img = ADJ ? nullptr : src + (long long)bc * WW;
  float* oimg = ADJ ? dst + (long long)bc * WW : nullptr;
  const float yv = ADJ ? __ldg(src + ((long long)bc * F.A + t) * F.D + j) * scale : 0.f;
  float acc = 0.f;
  for (int i = 0; i < F.G; ++i) {
    const float xi = lin_at(i, F.G, F.step_g);
    const float d = (F.half_len * (xi + F.src)) / F.den;
    const float y = yj * d;
    const float gx = fmaf(y, s, xi * c);
    const float gy = fmaf(y, c, -(xi * s));
    const float px = ((gx + 1.0f) * 0.5f) * gm1, py = ((gy + 1.0f) * 0.5f) * gm1;
    const float fx = floorf(px), fy = floorf(py);
    if (!(fx >= (float)(F.pb - 1) && fx < (float)(F.pb + F.W) && fy >= (float)(F.pb - 1) && fy < (float)(F.pb + F.W))) continue;
    const int X0 = (int)fx, Y0 = (int)fy;
    const float wx1 = px - fx, wy1 = py - fy, wx0 = (fx + 1.0f) - px, wy0 = (fy + 1.0f) - py;
    if (!ADJ) {
      const float v00 = img_at(img, R, X0, Y0), v01 = img_at(img, R, X0 + 1, Y0);
      const float v10 = img_at(img, R, X0, Y0 + 1), v11 = img_at(img, R, X0 + 1, Y0 + 1);
      acc += v00 * (wx0 * wy0) + v01 * (wx1 * wy0) + v10 * (wx0 * wy1) + v11 * (wx1 * wy1);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int X = X0 + (k & 1), Y = Y0 + (k >> 1);
        const int x = X - F.pb, yy = Y - F.pb;
        if (x < 0 || x >= F.W || yy < 0 || yy >= F.W) continue;
        if (F.circle) {
          const float ax = 2.0f * (float)x / (float)(F.W - 1) - 1.0f, ay = 2.0f * (float)yy / (float)(F.W - 1) - 1.0f;
          if (!(ax * ax + ay * ay <= 1.0f)) continue;
        }
        const float w = ((k & 1) ? wx1 : wx0) * ((k >> 1) ? wy1 : wy0);
        atomicAdd(oimg + (long long)yy * F.W + x, yv * w);
      }
    }
  }
  if (!ADJ) dst[((long long)bc * F.A + t) * F.D + j] = acc * scale;
}

static int make_geom(RadonGeom* G, int W, int P, int A, int circle) {
  if (W < 1 || P < W || A < 1) return set_error(DINVK_EINVAL, "radon: bad geometry W=%d P=%d A=%d", W, P, A);
  if (circle && P != W) return set_error(DINVK_EINVAL, "radon: circle=1 requires P == W");
  G->W = W; G->P = P; G->A = A; G->circle = circle ? 1 : 0;
  G->pb = circle ? 0 : (P / 2 - W / 2);  // (W + pad)//2 - W//2 with pad = P - W   (radon.py:262-266)
  G->step = P > 1 ? (1.0f - (-1.0f)) / (float)(P - 1) : 0.f;
  return 0;
}

}  // namespace dinvk

using namespace dinvk;

extern "C" int dinvk_radon_fwd(const float* x, float* sino, int BC, int W, int P, int A, int circle, const float* cos_t,
                               const float* sin_t, float scale, void* stream) {
  DINVK_CHECK_ARG(x && sino && cos_t && sin_t && BC >= 0, "dinvk_radon_fwd: bad arguments");
  RadonGeom G;
  int rc = make_geom(&G, W, P, A, circle);
  if (rc) return rc;
  if (BC == 0) return DINVK_OK;
  DINVK_CHECK_ARG(A <= 65535 && BC <= 65535, "dinvk_radon_fwd: grid too large");
  if (tiled_ok(x, W, A)) {
    rc = launch_tiled(false, x, nullptr, sino, BC, G, cos_t, sin_t, scale, stream);
    if (rc >= 0) return rc;
  }
  DINVK_LAUNCH(radon_fwd_kernel, dim3(ceil_div(P, 128), A, BC), dim3(128), 0, stream, x, sino, G, cos_t, sin_t, scale);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_radon_adj(const float* sino, float* x, int BC, int W, int P, int A, int circle, const float* cos_t,
                               const float* sin_t, float scale, void* stream) {
  DINVK_CHECK_ARG(x && sino && cos_t && sin_t && BC >= 0, "dinvk_radon_adj: bad arguments");
  RadonGeom G;
  int rc = make_geom(&G, W, P, A, circle);
  if (rc) return rc;
  if (BC == 0) return DINVK_OK;
  DINVK_CHECK_ARG(BC <= 65535 && A <= 4096, "dinvk_radon_adj: grid too large");
  if (tiled_ok(x, W, A)) {
    rc = launch_tiled(true, nullptr, sino, x, BC, G, cos_t, sin_t, scale, stream);
    if (rc >= 0) return rc;
  }
  // the Q45 tables: 2 A * 8 bytes, above the default 48 KB for A > 3072
  const size_t smem = 2 * (size_t)A * sizeof(long long);
  if ((rc = allow_smem(radon_adj_kernel, smem))) return rc;
  DINVK_LAUNCH(radon_adj_kernel, dim3(ceil_div((long long)W * W, 256), BC), dim3(256), smem, stream, sino, x, G, cos_t, sin_t, scale);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_iradon_bp(const float* sino, float* x, int BC, int W, int P, int A, int circle, const float* cos_t,
                               const float* sin_t, float scale, void* stream) {
  DINVK_CHECK_ARG(x && sino && cos_t && sin_t && BC >= 0, "dinvk_iradon_bp: bad arguments");
  RadonGeom G;
  int rc = make_geom(&G, W, P, A, circle);
  if (rc) return rc;
  if (BC == 0) return DINVK_OK;
  DINVK_CHECK_ARG(BC <= 65535 && A <= 4096, "dinvk_iradon_bp: grid too large");
  const size_t smem = 2 * (size_t)A * sizeof(float);
  if ((rc = allow_smem(iradon_bp_kernel, smem))) return rc;
  DINVK_LAUNCH(iradon_bp_kernel, dim3(ceil_div((long long)W * W, 256), BC), dim3(256), smem, stream, sino, x, G, cos_t, sin_t, scale);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_fanbeam(const float* in, float* out, int BC, int W, int G, int D, int A, int circle, const float* cos_t,
                             const float* sin_t, float half_len, float src, float den, float scale, int adjoint, void* stream) {
  DINVK_CHECK_ARG(in && out && cos_t && sin_t && BC >= 0, "dinvk_fanbeam: bad arguments");
  DINVK_CHECK_ARG(W >= 1 && G >= W && D >= 1 && A >= 1, "dinvk_fanbeam: bad geometry W=%d G=%d D=%d A=%d", W, G, D, A);
  DINVK_CHECK_ARG(!circle || G == W, "dinvk_fanbeam: circle=1 requires G == W");
  DINVK_CHECK_ARG(A <= 65535 && BC <= 65535, "dinvk_fanbeam: grid too large");
  if (BC == 0) return DINVK_OK;
  FanGeom F;
  F.W = W; F.G = G; F.D = D; F.A = A; F.circle = circle ? 1 : 0;
  F.pb = circle ? 0 : (G / 2 - W / 2);
  F.step_g = G > 1 ? 2.0f / (float)(G - 1) : 0.f;
  F.step_d = D > 1 ? 2.0f / (float)(D - 1) : 0.f;
  F.half_len = half_len; F.src = src; F.den = den;
  if (adjoint) {
    if (cudaMemsetAsync(out, 0, (size_t)BC * W * W * sizeof(float), (cudaStream_t)stream) != cudaSuccess)
      return set_error(DINVK_ECUDA, "dinvk_fanbeam: memset failed");
    DINVK_LAUNCH(fanbeam_kernel<true>, dim3(ceil_div(D, 128), A, BC), dim3(128), 0, stream, in, out, F, cos_t, sin_t, scale);
  } else {
    DINVK_LAUNCH(fanbeam_kernel<false>, dim3(ceil_div(D, 128), A, BC), dim3(128), 0, stream, in, out, F, cos_t, sin_t, scale);
  }
  return DINVK_POST_LAUNCH();
}
