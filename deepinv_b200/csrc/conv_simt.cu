// conv_simt.cu — fp32 (reference-precision) denoiser convolutions on CUDA cores, NCHW.
//
// Replaces the ATen calls behind deepinv/models/drunet.py:200-210,323-433 (3x3 conv, ResBlock,
// strided 2x2 down-conv, transposed 2x2 up-conv, all bias-free) and deepinv/models/dncnn.py:116-131
// (3x3 conv + bias + ReLU).  This is the parity path (matches the fp32 reference to ~1e-6); the
// throughput path is the wgmma implicit GEMM in conv_tc.cu.
//
//   kind 0: 3x3, stride 1, zero padding 1 — register-tiled direct convolution: a CTA computes an
//           8x32 pixel x 32 output-channel tile, staging 8 input channels (with halo) and their
//           weights in shared memory per step; each thread owns 4 pixels x 8 channels.
//   kind 1/2: 2x2 stride-2 conv / transposed conv as a small gather-GEMM-scatter (64x32 tiles).
// Fusions: input sum (x + xadd: the U-Net skip), bias, ReLU, residual add.
#include "common.cuh"
#ifndef DINVK_EMUL
#include <cstdlib>
#endif

namespace dinvk {

constexpr int C3_CC = 8;     // input channels per step
constexpr int C3_TH = 8;     // tile rows
constexpr int C3_TW = 32;    // tile cols
constexpr int C3_TC = 32;    // output channels per CTA
constexpr int C3_ROWP = 36;  // padded smem row (34 used)
constexpr int C3_WS = 36;    // padded weight row in shared memory (32 used): keeps float4 alignment, spreads the staging stores

constexpr int C3_IN_ELEMS = C3_CC * (C3_TH + 2) * (C3_TW + 2);  // staged inputs per chunk (8 x 10 x 34)
constexpr int C3_IN_IT = (C3_IN_ELEMS + 255) / 256;              // 11 per thread
constexpr int C3_W_IT = C3_CC * 9 * C3_TC / 256;                 // 9 per thread

// PF = true: software-pipelined staging — the global loads of chunk k+1 are issued into registers before the FMAs of chunk k
// and stored to shared memory after them, so their latency (ncu: long-scoreboard is the top stall of the synchronous version)
// is covered by the compute of the same CTA instead of only by the other resident CTAs.
template <bool PF>
__global__ void __launch_bounds__(256, PF ? 2 : 3) conv3x3_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                          const float* __restrict__ w, const float* __restrict__ bias,
                                                          const float* __restrict__ res, float* __restrict__ out,
                                                          int Cin, int Cout, int H, int W, int tiles_x, int act) {
  __shared__ __align__(16) float s_in[C3_CC][C3_TH + 2][C3_ROWP];
  __shared__ __align__(16) float s_w[C3_CC * 9][C3_WS];
  const int tid = threadIdx.x;
  const int tx = tid & 7, ty = (tid >> 3) & 7, tz = tid >> 6;
  const int ty0 = (blockIdx.x / tiles_x) * C3_TH, tx0 = (blockIdx.x % tiles_x) * C3_TW;
  const int co0 = blockIdx.y * C3_TC;
  const int b = blockIdx.z;
  const long long HW = (long long)H * W;
  const float* xb = x + (long long)b * Cin * HW;
  const float* ab = xadd ? xadd + (long long)b * Cin * HW : nullptr;

  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[p][q] = 0.f;

  // one staged input (halo, zero padding) / weight of chunk c0 for flat index idx
  auto load_in = [&](int c0, int idx) -> float {
    const int c = idx / ((C3_TH + 2) * (C3_TW + 2));
    const int rem = idx - c * ((C3_TH + 2) * (C3_TW + 2));
    const int r = rem / (C3_TW + 2), col = rem - r * (C3_TW + 2);
    const int gy = ty0 + r - 1, gx = tx0 + col - 1;
    float v = 0.f;
    if (idx < C3_IN_ELEMS && c0 + c < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const long long o = (long long)(c0 + c) * HW + (long long)gy * W + gx;
      v = __ldg(xb + o);
      if (ab) v += __ldg(ab + o);
    }
    return v;
  };
  // weights w[(co, ci, ky, kx)] go to s_w[(ci, tap)][co] (rows padded to C3_WS = 36 floats).  A warp covers 8 consecutive
  // (ci, tap) entries x 4 output channels: 32-byte global segments, and shared banks 4*(ci,tap) + co -> all 32 distinct
  auto load_w = [&](int c0, int idx, int& soff) -> float {
    const int blk = idx >> 5;
    const int ck = (blk % 9) * 8 + (idx & 7), co = (blk / 9) * 4 + ((idx >> 3) & 3);
    soff = ck * C3_WS + co;
    float v = 0.f;
    if (c0 + ck / 9 < Cin && co0 + co < Cout) v = __ldg(w + ((long long)(co0 + co) * Cin + c0) * 9 + ck);
    return v;
  };
  float* s_in_flat = &s_in[0][0][0];
  float* s_w_flat = &s_w[0][0];
  float rin[PF ? C3_IN_IT : 1], rw[PF ? C3_W_IT : 1];
  if (PF) {
#pragma unroll
    for (int it = 0; it < C3_IN_IT; ++it) rin[PF ? it : 0] = load_in(0, tid + 256 * it);
#pragma unroll
    for (int it = 0; it < C3_W_IT; ++it) { int so; rw[PF ? it : 0] = load_w(0, tid + 256 * it, so); }
  }

  for (int c0 = 0; c0 < Cin; c0 += C3_CC) {
    if (PF) {
      // registers of this chunk -> shared memory (row pitch 36 for 34 used columns: flat offset = idx + 2 * (idx / 34))
#pragma unroll
      for (int it = 0; it < C3_IN_IT; ++it) {
        const int idx = tid + 256 * it;
        if (idx < C3_IN_ELEMS) s_in_flat[idx + 2 * (idx / (C3_TW + 2))] = rin[PF ? it : 0];
      }
#pragma unroll
      for (int it = 0; it < C3_W_IT; ++it) {
        const int idx = tid + 256 * it, blk = idx >> 5;
        s_w_flat[((blk % 9) * 8 + (idx & 7)) * C3_WS + (blk / 9) * 4 + ((idx >> 3) & 3)] = rw[PF ? it : 0];
      }
      __syncthreads();
      if (c0 + C3_CC < Cin) {  // next chunk's loads fly during this chunk's FMAs
#pragma unroll
        for (int it = 0; it < C3_IN_IT; ++it) rin[PF ? it : 0] = load_in(c0 + C3_CC, tid + 256 * it);
#pragma unroll
        for (int it = 0; it < C3_W_IT; ++it) { int so; rw[PF ? it : 0] = load_w(c0 + C3_CC, tid + 256 * it, so); }
      }
    } else {
      for (int idx = tid; idx < C3_IN_ELEMS; idx += 256) s_in_flat[idx + 2 * (idx / (C3_TW + 2))] = load_in(c0, idx);
      for (int idx = tid; idx < C3_CC * 9 * C3_TC; idx += 256) {
        int so;
        const float v = load_w(c0, idx, so);
        s_w_flat[so] = v;
      }
      __syncthreads();
    }
#pragma unroll
    for (int c = 0; c < C3_CC; ++c) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const float4 i0 = *reinterpret_cast<const float4*>(&s_in[c][ty + ky][tx * 4]);
        const float2 i1 = *reinterpret_cast<const float2*>(&s_in[c][ty + ky][tx * 4 + 4]);
        const float in6[6] = {i0.x, i0.y, i0.z, i0.w, i1.x, i1.y};
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float4 w0 = *reinterpret_cast<const float4*>(&s_w[c * 9 + ky * 3 + kx][tz * 8]);
          const float4 w1 = *reinterpret_cast<const float4*>(&s_w[c * 9 + ky * 3 + kx][tz * 8 + 4]);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[p][q] = fmaf(in6[p + kx], wv[q], acc[p][q]);
        }
      }
    }
    __syncthreads();
  }

  // epilogue: bias -> activation -> residual
  const int gy = ty0 + ty;
  if (gy < H) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int co = co0 + tz * 8 + q;
      if (co < Cout) {
        const float bv = bias ? __ldg(bias + co) : 0.f;
        const long long ob = ((long long)b * Cout + co) * HW + (long long)gy * W;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int gx = tx0 + tx * 4 + p;
          if (gx < W) {
            float v = acc[p][q] + bv;
            if (act == 1) v = fmaxf(v, 0.f);
            if (res) v += __ldg(res + ob + gx);
            out[ob + gx] = v;
          }
        }
      }
    }
  }
}

// gather-GEMM-scatter for the 2x2 stride-2 conv (mode 1) and its transpose (mode 2)
//   mode 1: M = B*Ho*Wo, N = Cout, K = 4*Cin;  A(m,k) = x[b, c, 2yo+dy, 2xo+dx], Wt(k,n) = w[n*K + k]
//   mode 2: M = B*H*W,   N = 4*Cout, K = Cin;  A(m,k) = (x+xadd)[b, k, y, x],   Wt(k,n) = w[k*N + n],
//           out[b, n/4, 2y + (n%4)/2, 2x + n%2]
constexpr int G_TM = 64, G_TN = 32, G_TK = 32;

__global__ void __launch_bounds__(256) conv2x2_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                          const float* __restrict__ w, const float* __restrict__ bias,
                                                          const float* __restrict__ res, float* __restrict__ out,
                                                          int B, int Cin, int Cout, int H, int W, int mode, int act) {
  __shared__ float sA[G_TK][G_TM + 1];
  __shared__ float sW[G_TK][G_TN + 1];
  const int tid = threadIdx.x;
  const int Ho = H / 2, Wo = W / 2;
  const long long M = mode == 1 ? (long long)B * Ho * Wo : (long long)B * H * W;
  const int N = mode == 1 ? Cout : 4 * Cout;
  const int K = mode == 1 ? 4 * Cin : Cin;
  const long long m0 = (long long)blockIdx.x * G_TM;
  const int n0 = blockIdx.y * G_TN;
  const int tm = tid & 31, tn = tid >> 5;  // thread owns pixels {tm, tm+32} x channels {tn*4 .. tn*4+3}
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  const long long HW = (long long)H * W;

  for (int k0 = 0; k0 < K; k0 += G_TK) {
    for (int idx = tid; idx < G_TK * G_TM; idx += 256) {
      const int kk = idx / G_TM, mm = idx - kk * G_TM;
      const long long m = m0 + mm;
      const int k = k0 + kk;
      float v = 0.f;
      if (m < M && k < K) {
        if (mode == 1) {
          const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho);
          const long long bb = m / ((long long)Wo * Ho);
          const int c = k >> 2, dy = (k >> 1) & 1, dx = k & 1;
          const long long o = (bb * Cin + c) * HW + (long long)(2 * yo + dy) * W + (2 * xo + dx);
          v = __ldg(x + o);
          if (xadd) v += __ldg(xadd + o);
        } else {
          const long long bb = m / HW, p = m - bb * HW;
          const long long o = (bb * Cin + k) * HW + p;
          v = __ldg(x + o);
          if (xadd) v += __ldg(xadd + o);
        }
      }
      sA[kk][mm] = v;
    }
    for (int idx = tid; idx < G_TK * G_TN; idx += 256) {
      int kk, nn;
      if (mode == 1) { nn = idx / G_TK; kk = idx - nn * G_TK; }  // k fastest in memory
      else { kk = idx / G_TN; nn = idx - kk * G_TN; }            // n fastest in memory
      const int k = k0 + kk, n = n0 + nn;
      float v = 0.f;
      if (k < K && n < N) v = mode == 1 ? __ldg(w + (long long)n * K + k) : __ldg(w + (long long)k * N + n);
      sW[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < G_TK; ++kk) {
      const float a0 = sA[kk][tm], a1 = sA[kk][tm + 32];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float wv = sW[kk][tn * 4 + q];
        acc[0][q] = fmaf(a0, wv, acc[0][q]);
        acc[1][q] = fmaf(a1, wv, acc[1][q]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long m = m0 + tm + 32 * i;
    if (m >= M) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = n0 + tn * 4 + q;
      if (n >= N) continue;
      long long o;
      int co;
      if (mode == 1) {
        const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho);
        const long long bb = m / ((long long)Wo * Ho);
        co = n;
        o = (bb * Cout + co) * ((long long)Ho * Wo) + (long long)yo * Wo + xo;
      } else {
        const long long bb = m / HW, p = m - bb * HW;
        const int y = (int)(p / W), xx = (int)(p - (long long)y * W);
        co = n >> 2;
        const int dy = (n >> 1) & 1, dx = n & 1;
        o = (bb * Cout + co) * (4 * HW) + (long long)(2 * y + dy) * (2 * W) + (2 * xx + dx);
      }
      float v = acc[i][q] + (bias ? __ldg(bias + co) : 0.f);
      if (act == 1) v = fmaxf(v, 0.f);
      if (res) v += __ldg(res + o);
      out[o] = v;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// 3-D (NCDHW) forward kernels for DRUNet(dim=3) (deepinv/models/drunet.py with Conv3d / ConvTranspose3d).
//   3x3x3: the 2-D kernel's CTA (8 x 32 pixels of ONE depth plane x 32 output channels) walks the three input planes z - 1 ..
//          z + 1 inside each 8-channel step; a plane outside the volume is the zero padding and is skipped.
//   2x2x2 stride 2 and its transpose: the 2-D gather-GEMM-scatter with 8 taps.
// Every offset is 64-bit: one 64-channel activation of a 64 x 256 x 256 volume is 2^28 elements.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 2) conv3x3x3_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                               const float* __restrict__ w, const float* __restrict__ bias,
                                                               const float* __restrict__ res, float* __restrict__ out, int Cin,
                                                               int Cout, int D, int H, int W, int tiles_x, int tiles, int act) {
  __shared__ __align__(16) float s_in[C3_CC][C3_TH + 2][C3_ROWP];
  __shared__ __align__(16) float s_w[C3_CC * 9][C3_WS];
  const int tid = threadIdx.x;
  const int tx = tid & 7, ty = (tid >> 3) & 7, tz = tid >> 6;
  const long long plane = blockIdx.x / tiles;   // b * D + z
  const int t = (int)(blockIdx.x - plane * tiles);
  const int ty0 = (t / tiles_x) * C3_TH, tx0 = (t % tiles_x) * C3_TW;
  const int co0 = blockIdx.y * C3_TC;
  const long long b = plane / D;
  const int z = (int)(plane - b * D);
  const long long HW = (long long)H * W, DHW = HW * D;
  const float* xb = x + b * Cin * DHW;
  const float* ab = xadd ? xadd + b * Cin * DHW : nullptr;

  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[p][q] = 0.f;
  float* s_in_flat = &s_in[0][0][0];
  float* s_w_flat = &s_w[0][0];

  for (int c0 = 0; c0 < Cin; c0 += C3_CC) {
    for (int kz = 0; kz < 3; ++kz) {
      const int zz = z + kz - 1;
      if (zz < 0 || zz >= D) continue;   // CTA-uniform
      for (int idx = tid; idx < C3_IN_ELEMS; idx += 256) {
        const int c = idx / ((C3_TH + 2) * (C3_TW + 2));
        const int rem = idx - c * ((C3_TH + 2) * (C3_TW + 2));
        const int r = rem / (C3_TW + 2), col = rem - r * (C3_TW + 2);
        const int gy = ty0 + r - 1, gx = tx0 + col - 1;
        float v = 0.f;
        if (c0 + c < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W) {
          const long long o = (long long)(c0 + c) * DHW + (long long)zz * HW + (long long)gy * W + gx;
          v = __ldg(xb + o);
          if (ab) v += __ldg(ab + o);
        }
        s_in_flat[idx + 2 * (idx / (C3_TW + 2))] = v;
      }
      // w[(co, ci, kz, ky, kx)] -> s_w[(ci, ky * 3 + kx)][co], the 2-D kernel's staging order
      for (int idx = tid; idx < C3_CC * 9 * C3_TC; idx += 256) {
        const int blk = idx >> 5;
        const int ck = (blk % 9) * 8 + (idx & 7), co = (blk / 9) * 4 + ((idx >> 3) & 3);
        const int ci = ck / 9, tap = ck - ci * 9;
        float v = 0.f;
        if (c0 + ci < Cin && co0 + co < Cout) v = __ldg(w + (((long long)(co0 + co) * Cin + c0 + ci) * 3 + kz) * 9 + tap);
        s_w_flat[ck * C3_WS + co] = v;
      }
      __syncthreads();
#pragma unroll
      for (int c = 0; c < C3_CC; ++c) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          const float4 i0 = *reinterpret_cast<const float4*>(&s_in[c][ty + ky][tx * 4]);
          const float2 i1 = *reinterpret_cast<const float2*>(&s_in[c][ty + ky][tx * 4 + 4]);
          const float in6[6] = {i0.x, i0.y, i0.z, i0.w, i1.x, i1.y};
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const float4 w0 = *reinterpret_cast<const float4*>(&s_w[c * 9 + ky * 3 + kx][tz * 8]);
            const float4 w1 = *reinterpret_cast<const float4*>(&s_w[c * 9 + ky * 3 + kx][tz * 8 + 4]);
            const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
            for (int p = 0; p < 4; ++p)
#pragma unroll
              for (int q = 0; q < 8; ++q) acc[p][q] = fmaf(in6[p + kx], wv[q], acc[p][q]);
          }
        }
      }
      __syncthreads();
    }
  }

  const int gy = ty0 + ty;
  if (gy < H) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int co = co0 + tz * 8 + q;
      if (co < Cout) {
        const float bv = bias ? __ldg(bias + co) : 0.f;
        const long long ob = ((b * Cout + co) * D + z) * HW + (long long)gy * W;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const int gx = tx0 + tx * 4 + p;
          if (gx < W) {
            float v = acc[p][q] + bv;
            if (act == 1) v = fmaxf(v, 0.f);
            if (res) v += __ldg(res + ob + gx);
            out[ob + gx] = v;
          }
        }
      }
    }
  }
}

// gather-GEMM-scatter for the 2x2x2 stride-2 conv (mode 1) and its transpose (mode 2), tap = dz * 4 + dy * 2 + dx
//   mode 1: M = B*Do*Ho*Wo, N = Cout, K = 8*Cin;  A(m,k) = (x+xadd)[b, k/8, 2zo+dz, 2yo+dy, 2xo+dx],  Wt(k,n) = w[n*K + k]
//   mode 2: M = B*D*H*W,    N = 8*Cout, K = Cin;  A(m,k) = (x+xadd)[b, k, z, y, x],  Wt(k,n) = w[k*N + n],
//           out[b, n/8, 2z+dz, 2y+dy, 2x+dx]
__global__ void __launch_bounds__(256) conv2x2x2_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                            const float* __restrict__ w, const float* __restrict__ bias,
                                                            const float* __restrict__ res, float* __restrict__ out,
                                                            int B, int Cin, int Cout, int D, int H, int W, int mode, int act) {
  __shared__ float sA[G_TK][G_TM + 1];
  __shared__ float sW[G_TK][G_TN + 1];
  const int tid = threadIdx.x;
  const int Do = D / 2, Ho = H / 2, Wo = W / 2;
  const long long HW = (long long)H * W, DHW = HW * D, OV = (long long)Do * Ho * Wo;
  const long long M = mode == 1 ? (long long)B * OV : (long long)B * DHW;
  const int N = mode == 1 ? Cout : 8 * Cout;
  const int K = mode == 1 ? 8 * Cin : Cin;
  const long long m0 = (long long)blockIdx.x * G_TM;
  const int n0 = blockIdx.y * G_TN;
  const int tm = tid & 31, tn = tid >> 5;
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};

  for (int k0 = 0; k0 < K; k0 += G_TK) {
    for (int idx = tid; idx < G_TK * G_TM; idx += 256) {
      const int kk = idx / G_TM, mm = idx - kk * G_TM;
      const long long m = m0 + mm;
      const int k = k0 + kk;
      float v = 0.f;
      if (m < M && k < K) {
        long long o;
        if (mode == 1) {
          const long long bb = m / OV, p = m - bb * OV;
          const int xo = (int)(p % Wo), yo = (int)((p / Wo) % Ho), zo = (int)(p / ((long long)Wo * Ho));
          const int c = k >> 3, dz = (k >> 2) & 1, dy = (k >> 1) & 1, dx = k & 1;
          o = (bb * Cin + c) * DHW + (long long)(2 * zo + dz) * HW + (long long)(2 * yo + dy) * W + (2 * xo + dx);
        } else {
          const long long bb = m / DHW, p = m - bb * DHW;
          o = (bb * Cin + k) * DHW + p;
        }
        v = __ldg(x + o);
        if (xadd) v += __ldg(xadd + o);
      }
      sA[kk][mm] = v;
    }
    for (int idx = tid; idx < G_TK * G_TN; idx += 256) {
      int kk, nn;
      if (mode == 1) { nn = idx / G_TK; kk = idx - nn * G_TK; }
      else { kk = idx / G_TN; nn = idx - kk * G_TN; }
      const int k = k0 + kk, n = n0 + nn;
      float v = 0.f;
      if (k < K && n < N) v = mode == 1 ? __ldg(w + (long long)n * K + k) : __ldg(w + (long long)k * N + n);
      sW[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < G_TK; ++kk) {
      const float a0 = sA[kk][tm], a1 = sA[kk][tm + 32];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float wv = sW[kk][tn * 4 + q];
        acc[0][q] = fmaf(a0, wv, acc[0][q]);
        acc[1][q] = fmaf(a1, wv, acc[1][q]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long m = m0 + tm + 32 * i;
    if (m >= M) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = n0 + tn * 4 + q;
      if (n >= N) continue;
      long long o;
      int co;
      if (mode == 1) {
        const long long bb = m / OV, p = m - bb * OV;
        co = n;
        o = (bb * Cout + co) * OV + p;
      } else {
        const long long bb = m / DHW, p = m - bb * DHW;
        const int z = (int)(p / HW), y = (int)((p - z * HW) / W), xx = (int)(p - z * HW - (long long)y * W);
        co = n >> 3;
        const int dz = (n >> 2) & 1, dy = (n >> 1) & 1, dx = n & 1;
        o = (bb * Cout + co) * (8 * DHW) + (long long)(2 * z + dz) * (4 * HW) + (long long)(2 * y + dy) * (2 * W) + (2 * xx + dx);
      }
      float v = acc[i][q] + (bias ? __ldg(bias + co) : 0.f);
      if (act == 1) v = fmaxf(v, 0.f);
      if (res) v += __ldg(res + o);
      out[o] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Backward kernels of the fp32 path (training through the denoiser: unfolded / DEQ models,
// deepinv/unfolded/unfolded.py:9-120, deep_equilibrium.py:70-139 — SURVEY §8(f) item 2).
// Data gradients reuse the forward kernels (a 3x3 convolution with the transposed, flipped filter;
// kind 1 <-> kind 2 for the 2x2 pair).  What is new is the weight gradient:
//   kind 0:  dw[co,ci,ky,kx] = sum_{b,y,x} g[b,co,y,x] * xin[b,ci,y+ky-1,x+kx-1]
// A CTA owns one 8-row band of one image, 32 output channels and 8 input channels; it walks the
// band tile by tile with the forward kernel's staging (input halo tile + the matching 8x32x32
// block of g, channel-fastest so that a thread reads its 4 output channels as one float4).  Thread
// = (4 output channels, 1 input channel, 2 of the 8 rows): 36 accumulators; 4 columns per step from a
// 3x6 register patch (float4 + float2 per row) and four float4 of g -> 144 FMAs per 10 shared loads.  The 4 row groups are
// summed through shared memory and leave as one atomicAdd per weight per CTA; the bias gradient
// (sum of g) rides along in the CTAs of input-channel chunk 0.
constexpr int WG_CI = 8;   // input channels per CTA
constexpr int WG_CO = 32;  // output channels per CTA
constexpr int WG_GS = 36;  // shared row of the g tile (32 channels + 4 pad)

template <int MINB>  // CTAs per SM the register allocation is held to (2: 119 registers; 3: 80 registers, 20 B of spills)
__global__ void __launch_bounds__(256, MINB) conv3x3_wgrad_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                                const float* __restrict__ g, float* __restrict__ dw,
                                                                float* __restrict__ dbias, int Cin, int Cout, int H, int W,
                                                                int tiles_x, int nci) {
  __shared__ __align__(16) float s_in[WG_CI][C3_TH + 2][C3_ROWP];
  __shared__ __align__(16) float s_g[C3_TH * C3_TW * WG_GS];  // [row][col][co (+4 pad)]; reused for the final reduction
  const int tid = threadIdx.x;
  const int lane64 = tid & 63, rg = tid >> 6;
  const int cg = lane64 & 7, ci = lane64 >> 3;
  const int ty0 = blockIdx.x * C3_TH;
  const int co0 = blockIdx.y * WG_CO;
  const int b = blockIdx.z / nci, c0 = (blockIdx.z % nci) * WG_CI;
  const long long HW = (long long)H * W;
  const float* xb = x + (long long)b * Cin * HW;
  const float* ab = xadd ? xadd + (long long)b * Cin * HW : nullptr;
  const float* gb = g + (long long)b * Cout * HW;
  const bool cta_bias = dbias != nullptr && c0 == 0;  // CTA-uniform: the bias gradient rides in the chunk-0 CTAs only
  const bool do_bias = cta_bias && ci == 0;

  float acc[4][9];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[q][k] = 0.f;
  float bsum[4] = {0.f, 0.f, 0.f, 0.f};

  for (int t = 0; t < tiles_x; ++t) {
    const int tx0 = t * C3_TW;
    for (int idx = tid; idx < WG_CI * (C3_TH + 2) * (C3_TW + 2); idx += 256) {
      const int c = idx / ((C3_TH + 2) * (C3_TW + 2));
      const int rem = idx - c * ((C3_TH + 2) * (C3_TW + 2));
      const int r = rem / (C3_TW + 2), col = rem - r * (C3_TW + 2);
      const int gy = ty0 + r - 1, gx = tx0 + col - 1;
      float v = 0.f;
      if (c0 + c < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W) {
        const long long o = (long long)(c0 + c) * HW + (long long)gy * W + gx;
        v = __ldg(xb + o);
        if (ab) v += __ldg(ab + o);
      }
      s_in[c][r][col] = v;
    }
    // g tile, channel-fastest with rows of WG_GS = 36 floats.  A warp covers 8 consecutive pixels x 4 channels: 32-byte global
    // segments, shared banks 4*pixel + channel -> all 32 distinct (a plain [pixel][32] layout filled pixel-fastest is a 32-way
    // bank conflict on every store: measured 2x the kernel's whole compute-phase shared traffic)
    for (int idx = tid; idx < WG_CO * C3_TH * C3_TW; idx += 256) {
      const int blk = idx >> 5;
      const int pix = (blk & 31) * 8 + (idx & 7), co = (blk >> 5) * 4 + ((idx >> 3) & 3);
      const int r = pix / C3_TW, col = pix - r * C3_TW;
      const int gy = ty0 + r, gx = tx0 + col;
      float v = 0.f;
      if (co0 + co < Cout && gy < H && gx < W) v = __ldg(gb + (long long)(co0 + co) * HW + (long long)gy * W + gx);
      s_g[pix * WG_GS + co] = v;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = rg * 2 + rr;
      // 4 output columns at a time: the 3 x 6 input patch they need comes in as one float4 + one float2 per row (compile-time
      // indexed from then on: no window shifting), the 4 x 4 block of g as four float4 -> 10 shared loads per 144 FMAs
#pragma unroll 2
      for (int c4 = 0; c4 < C3_TW; c4 += 4) {
        float in[3][6];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          const float4 i0 = *reinterpret_cast<const float4*>(&s_in[ci][r + ky][c4]);
          const float2 i1 = *reinterpret_cast<const float2*>(&s_in[ci][r + ky][c4 + 4]);
          in[ky][0] = i0.x; in[ky][1] = i0.y; in[ky][2] = i0.z; in[ky][3] = i0.w; in[ky][4] = i1.x; in[ky][5] = i1.y;
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float4 g4 = *reinterpret_cast<const float4*>(&s_g[(r * C3_TW + c4 + p) * WG_GS + cg * 4]);
          const float gv[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if (cta_bias) bsum[q] += gv[q];
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
              for (int kx = 0; kx < 3; ++kx) acc[q][ky * 3 + kx] = fmaf(gv[q], in[ky][p + kx], acc[q][ky * 3 + kx]);
          }
        }
      }
    }
    __syncthreads();
  }

  // sum the 4 row groups: groups 2,3 -> smem -> groups 0,1 ; group 1 -> smem -> group 0
  float* red = s_g;  // 2 * 64 * 40 floats <= 9216
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    const int half = round == 0 ? 2 : 1;
    if (rg >= half && rg < 2 * half) {
      float* dst = red + ((rg - half) * 64 + lane64) * 40;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int k = 0; k < 9; ++k) dst[q * 9 + k] = acc[q][k];
        dst[36 + q] = bsum[q];
      }
    }
    __syncthreads();
    if (rg < half) {
      const float* src = red + (rg * 64 + lane64) * 40;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[q][k] += src[q * 9 + k];
        bsum[q] += src[36 + q];
      }
    }
    __syncthreads();
  }
  if (rg == 0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int co = co0 + cg * 4 + q;
      if (co >= Cout) continue;
      if (c0 + ci < Cin) {
        float* d = dw + ((long long)co * Cin + (c0 + ci)) * 9;
#pragma unroll
        for (int k = 0; k < 9; ++k) atomicAdd(d + k, acc[q][k]);
      }
      if (do_bias) atomicAdd(dbias + co, bsum[q]);
    }
  }
}

// weight gradient of the 2x2 pair as D[k][n] = sum_m A(m,k) * G(m,n) with the forward kernel's gathers:
//   mode 1: A(m,k) = (x+xadd)[b, k/4, 2yo + (k/2)%2, 2xo + k%2],  G(m,n) = g[b, n, yo, xo],          dw[n*K + k]
//   mode 2: A(m,k) = (x+xadd)[b, k, y, x],                        G(m,n) = g[b, n/4, 2y+(n/2)%2, 2x+n%2],  dw[k*N + n]
// CTA = 32x32 block of D over a chunk of WG2_MCHUNK rows m; thread = 2x2 outputs; one atomicAdd per output.
constexpr int WG2_MCHUNK = 4096;

__global__ void __launch_bounds__(256) conv2x2_wgrad_f32_kernel(const float* __restrict__ x, const float* __restrict__ xadd,
                                                                const float* __restrict__ g, float* __restrict__ dw,
                                                                float* __restrict__ dbias, int B, int Cin, int Cout, int H,
                                                                int W, int mode) {
  __shared__ float sA[G_TM][32 + 1];
  __shared__ float sG[G_TM][32 + 1];
  const int tid = threadIdx.x;
  const int Ho = H / 2, Wo = W / 2;
  const long long M = mode == 1 ? (long long)B * Ho * Wo : (long long)B * H * W;
  const int N = mode == 1 ? Cout : 4 * Cout;
  const int K = mode == 1 ? 4 * Cin : Cin;
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
  const long long mbeg = (long long)blockIdx.z * WG2_MCHUNK;
  const long long mend = mbeg + WG2_MCHUNK < M ? mbeg + WG2_MCHUNK : M;
  const int tk = (tid & 15) * 2, tn = (tid >> 4) * 2;
  const long long HW = (long long)H * W;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float bs = 0.f;  // bias gradient: thread tid < 32 of the k-block 0 sums column n0 + tid (mode 1 only)

  for (long long m0 = mbeg; m0 < mend; m0 += G_TM) {
    for (int idx = tid; idx < G_TM * 32; idx += 256) {
      const int mm = idx & (G_TM - 1), kk = idx / G_TM;  // m fastest: coalesced along pixels
      const long long m = m0 + mm;
      const int k = k0 + kk;
      float v = 0.f;
      if (m < mend && k < K) {
        long long o;
        if (mode == 1) {
          const int xo = (int)(m % Wo), yo = (int)((m / Wo) % Ho);
          const long long bb = m / ((long long)Wo * Ho);
          const int c = k >> 2, dy = (k >> 1) & 1, dx = k & 1;
          o = (bb * Cin + c) * HW + (long long)(2 * yo + dy) * W + (2 * xo + dx);
        } else {
          const long long bb = m / HW, p = m - bb * HW;
          o = (bb * Cin + k) * HW + p;
        }
        v = __ldg(x + o);
        if (xadd) v += __ldg(xadd + o);
      }
      sA[mm][kk] = v;
    }
    for (int idx = tid; idx < G_TM * 32; idx += 256) {
      const int mm = idx & (G_TM - 1), nn = idx / G_TM;
      const long long m = m0 + mm;
      const int n = n0 + nn;
      float v = 0.f;
      if (m < mend && n < N) {
        if (mode == 1) {
          const long long bb = m / ((long long)Wo * Ho), p = m - bb * ((long long)Wo * Ho);
          v = __ldg(g + (bb * Cout + n) * ((long long)Ho * Wo) + p);
        } else {
          const long long bb = m / HW, p = m - bb * HW;
          const int y = (int)(p / W), xx = (int)(p - (long long)y * W);
          const int co = n >> 2, dy = (n >> 1) & 1, dx = n & 1;
          v = __ldg(g + (bb * Cout + co) * (4 * HW) + (long long)(2 * y + dy) * (2 * W) + (2 * xx + dx));
        }
      }
      sG[mm][nn] = v;
    }
    __syncthreads();
#pragma unroll 8
    for (int mm = 0; mm < G_TM; ++mm) {
      const float a0 = sA[mm][tk], a1 = sA[mm][tk + 1];
      const float g0 = sG[mm][tn], g1 = sG[mm][tn + 1];
      acc[0][0] = fmaf(a0, g0, acc[0][0]);
      acc[0][1] = fmaf(a0, g1, acc[0][1]);
      acc[1][0] = fmaf(a1, g0, acc[1][0]);
      acc[1][1] = fmaf(a1, g1, acc[1][1]);
    }
    if (dbias && blockIdx.x == 0 && tid < 32)
      for (int mm = 0; mm < G_TM; ++mm) bs += sG[mm][tid];
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int k = k0 + tk + i, n = n0 + tn + j;
      if (k < K && n < N) atomicAdd(dw + (mode == 1 ? (long long)n * K + k : (long long)k * N + n), acc[i][j]);
    }
  if (dbias && blockIdx.x == 0 && tid < 32 && n0 + tid < N) atomicAdd(dbias + (mode == 1 ? n0 + tid : (n0 + tid) >> 2), bs);
}

// g_in = g * [out > 0]  (backward of the ReLU fused into the forward launch; `out` is the forward's output)
__global__ void __launch_bounds__(256) relu_bwd_kernel(const float* __restrict__ g, const float* __restrict__ out,
                                                       float* __restrict__ gin, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    gin[i] = out[i] > 0.f ? g[i] : 0.f;
}

}  // namespace dinvk

using namespace dinvk;

extern "C" int dinvk_conv_f32(const float* x, const float* xadd, const float* weight, const float* bias, const float* res,
                              float* out, int B, int Cin, int Cout, int H, int W, int kind, int act, void* stream) {
  DINVK_CHECK_ARG(x && weight && out, "dinvk_conv_f32: null pointer");
  DINVK_CHECK_ARG(B >= 0 && Cin >= 1 && Cout >= 1 && H >= 1 && W >= 1, "dinvk_conv_f32: bad shape");
  DINVK_CHECK_ARG(kind >= 0 && kind <= 2, "dinvk_conv_f32: kind %d", kind);
  DINVK_CHECK_ARG(act == 0 || act == 1, "dinvk_conv_f32: act %d", act);
  if (B == 0) return DINVK_OK;
  if (kind == 0) {
    const int tiles_x = ceil_div(W, C3_TW), tiles_y = ceil_div(H, C3_TH);
    DINVK_CHECK_ARG(B <= 65535 && ceil_div(Cout, C3_TC) <= 65535, "dinvk_conv_f32: grid too large");
    static const bool prefetch = getenv("DINVK_F32_PREFETCH") ? atoi(getenv("DINVK_F32_PREFETCH")) != 0 : false;
    if (prefetch)
      DINVK_LAUNCH(conv3x3_f32_kernel<true>, dim3(tiles_x * tiles_y, ceil_div(Cout, C3_TC), B), dim3(256), 0, stream, x, xadd,
                   weight, bias, res, out, Cin, Cout, H, W, tiles_x, act);
    else
      DINVK_LAUNCH(conv3x3_f32_kernel<false>, dim3(tiles_x * tiles_y, ceil_div(Cout, C3_TC), B), dim3(256), 0, stream, x, xadd,
                   weight, bias, res, out, Cin, Cout, H, W, tiles_x, act);
  } else {
    if (kind == 1) DINVK_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "dinvk_conv_f32: strided conv needs even H, W");
    const long long M = kind == 1 ? (long long)B * (H / 2) * (W / 2) : (long long)B * H * W;
    const int N = kind == 1 ? Cout : 4 * Cout;
    DINVK_LAUNCH(conv2x2_f32_kernel, dim3((unsigned)ceil_div(M, G_TM), ceil_div(N, G_TN)), dim3(256), 0, stream, x, xadd,
                 weight, bias, res, out, B, Cin, Cout, H, W, kind, act);
  }
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_conv3d_f32(const float* x, const float* xadd, const float* weight, const float* bias, const float* res,
                                float* out, int B, int Cin, int Cout, int D, int H, int W, int kind, int act, void* stream) {
  DINVK_CHECK_ARG(x && weight && out, "dinvk_conv3d_f32: null pointer");
  DINVK_CHECK_ARG(B >= 0 && Cin >= 1 && Cout >= 1 && D >= 1 && H >= 1 && W >= 1, "dinvk_conv3d_f32: bad shape");
  DINVK_CHECK_ARG(kind >= 0 && kind <= 2, "dinvk_conv3d_f32: kind %d not in 0..2", kind);
  DINVK_CHECK_ARG(act == 0 || act == 1, "dinvk_conv3d_f32: act %d", act);
  DINVK_CHECK_ARG(kind != 1 || (D % 2 == 0 && H % 2 == 0 && W % 2 == 0), "dinvk_conv3d_f32: strided conv needs even D, H, W (got %d, %d, %d)",
                  D, H, W);
  // the transposed conv's output is the largest tensor of a call: 8 voxels per input voxel
  DINVK_CHECK_ARG(product_fits(B, Cin > Cout ? Cin : Cout, D, H, W, 8, 4), "dinvk_conv3d_f32: volume (%d, %d, %d, %d, %d) too large", B,
                  Cin > Cout ? Cin : Cout, D, H, W);
  if (B == 0) return DINVK_OK;
  if (kind == 0) {
    const int tiles_x = ceil_div(W, C3_TW), tiles = tiles_x * ceil_div(H, C3_TH);
    DINVK_CHECK_ARG((long long)tiles * D * B < (1LL << 31) && ceil_div(Cout, C3_TC) <= 65535, "dinvk_conv3d_f32: grid too large");
    DINVK_LAUNCH(conv3x3x3_f32_kernel, dim3((unsigned)((long long)tiles * D * B), ceil_div(Cout, C3_TC)), dim3(256), 0, stream, x, xadd,
                 weight, bias, res, out, Cin, Cout, D, H, W, tiles_x, tiles, act);
  } else {
    const long long M = kind == 1 ? (long long)B * (D / 2) * (H / 2) * (W / 2) : (long long)B * D * H * W;
    const int N = kind == 1 ? Cout : 8 * Cout;
    DINVK_CHECK_ARG((M + G_TM - 1) / G_TM < (1LL << 31) && ceil_div(N, G_TN) <= 65535, "dinvk_conv3d_f32: grid too large");
    DINVK_LAUNCH(conv2x2x2_f32_kernel, dim3((unsigned)((M + G_TM - 1) / G_TM), ceil_div(N, G_TN)), dim3(256), 0, stream, x, xadd,
                 weight, bias, res, out, B, Cin, Cout, D, H, W, kind, act);
  }
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_conv_f32_wgrad(const float* x, const float* xadd, const float* gout, float* dweight, float* dbias,
                                    int B, int Cin, int Cout, int H, int W, int kind, void* stream) {
  DINVK_CHECK_ARG(x && gout && dweight, "dinvk_conv_f32_wgrad: null pointer");
  DINVK_CHECK_ARG(B >= 0 && Cin >= 1 && Cout >= 1 && H >= 1 && W >= 1, "dinvk_conv_f32_wgrad: bad shape");
  DINVK_CHECK_ARG(kind >= 0 && kind <= 2, "dinvk_conv_f32_wgrad: kind %d", kind);
  const size_t wn = (size_t)Cout * Cin * (kind == 0 ? 9 : 4);
  if (cudaMemsetAsync(dweight, 0, wn * sizeof(float), (cudaStream_t)stream) != cudaSuccess)
    return set_error(DINVK_ECUDA, "dinvk_conv_f32_wgrad: memset failed");
  if (dbias && cudaMemsetAsync(dbias, 0, (size_t)Cout * sizeof(float), (cudaStream_t)stream) != cudaSuccess)
    return set_error(DINVK_ECUDA, "dinvk_conv_f32_wgrad: memset failed");
  if (B == 0) return DINVK_OK;
  if (kind == 0) {
    const int tiles_x = ceil_div(W, C3_TW), tiles_y = ceil_div(H, C3_TH), nci = ceil_div(Cin, WG_CI);
    DINVK_CHECK_ARG((long long)B * nci <= 65535 && ceil_div(Cout, WG_CO) <= 65535, "dinvk_conv_f32_wgrad: grid too large");
    static const int occ = getenv("DINVK_WGRAD_OCC") ? atoi(getenv("DINVK_WGRAD_OCC")) : 2;
    if (occ == 3)
      DINVK_LAUNCH(conv3x3_wgrad_f32_kernel<3>, dim3(tiles_y, ceil_div(Cout, WG_CO), B * nci), dim3(256), 0, stream, x, xadd, gout,
                   dweight, dbias, Cin, Cout, H, W, tiles_x, nci);
    else
      DINVK_LAUNCH(conv3x3_wgrad_f32_kernel<2>, dim3(tiles_y, ceil_div(Cout, WG_CO), B * nci), dim3(256), 0, stream, x, xadd, gout,
                   dweight, dbias, Cin, Cout, H, W, tiles_x, nci);
  } else {
    if (kind == 1) DINVK_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "dinvk_conv_f32_wgrad: strided conv needs even H, W");
    const long long M = kind == 1 ? (long long)B * (H / 2) * (W / 2) : (long long)B * H * W;
    const int N = kind == 1 ? Cout : 4 * Cout, K = kind == 1 ? 4 * Cin : Cin;
    DINVK_CHECK_ARG(ceil_div(M, WG2_MCHUNK) <= 65535, "dinvk_conv_f32_wgrad: grid too large");
    DINVK_LAUNCH(conv2x2_wgrad_f32_kernel, dim3(ceil_div(K, 32), ceil_div(N, 32), (unsigned)ceil_div(M, WG2_MCHUNK)), dim3(256),
                 0, stream, x, xadd, gout, dweight, dbias, B, Cin, Cout, H, W, kind);
  }
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_relu_bwd(const float* gout, const float* out, float* gin, long long n, void* stream) {
  DINVK_CHECK_ARG(gout && out && gin && n >= 0, "dinvk_relu_bwd: bad argument");
  if (n == 0) return DINVK_OK;
  const long long want = (n + 255) / 256;
  const int grid = (int)(want < 148 * 16 ? want : 148 * 16);
  DINVK_LAUNCH(relu_bwd_kernel, dim3(grid), dim3(256), 0, stream, gout, out, gin, n);
  return DINVK_POST_LAUNCH();
}
