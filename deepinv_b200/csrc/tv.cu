// tv.cu — total-variation and TGV proxes (over-relaxed Chambolle-Pock, temporally blocked) and their stencils.
//
// Replaces
//   TVDenoiser.forward / TVL1Denoiser         deepinv/models/tv.py:86-151, 238-239
//   TVDenoiser.nabla / nabla_adjoint          deepinv/models/tv.py:153-218 (2-D)
//   TGVDenoiser.forward                       deepinv/models/tgv.py:93-213 (2-D)
//   TGVDenoiser.epsilon / epsilon_adjoint     deepinv/models/tgv.py:229-312 (2-D)
//   TVPrior.fn / grad, TVL1Prior.fn           deepinv/optim/prior.py:507-572, 595-611
//
// Both proxes run on one scaffold.  A CP kernel runs up to K iterations per launch; each CTA owns a T x T tile of one
// (b, c) plane and stages the region HALO pixels wider on every side (Tile).  The fields each pixel only reads at itself
// stay in the owning thread's registers for the whole launch, the fields a stencil reads at neighbours in shared memory.
// A stencil pass is only valid on a band of the region that shrinks by one pixel per side per stencil, so each pass runs
// over its own band (for_region) and after K iterations exactly the T x T core is valid and only it is written back.
// Every pixel is the same formula on the same inputs whatever T and K are, so the choice of T and K changes no output bit.
// The launch protocol is shared too: the control block at the head of the workspace says where the solve stands
// (begin_launch), and the last CTA of a launch applies the reference's break test and writes it back (finish_launch).
//
//   tv_cp_kernel    one stencil deep per iteration (nabla_adjoint, then nabla): HALO = K, region (T + 2K)^2.
//   tgv_cp_kernel   two stencils deep (epsilon_adjoint, nabla_adjoint, nabla, epsilon): HALO = 2K, region (T + 4K)^2.
//
// The four operators are written once over an accessor (nabla, nabla_adjoint, epsilon, epsilon_adjoint); the CP kernels
// apply them to shared memory and the standalone stencil kernels to global memory.  Every arithmetic step is rounded
// separately (__fmul_rn / __fadd_rn: no FMA contraction) in the reference's order, so the iterate follows the fp32 torch
// loop operation by operation.
#include "common.cuh"

#ifndef DINVK_TV_TILE
#define DINVK_TV_TILE 56
#endif
#ifndef DINVK_TV_BLOCK
#define DINVK_TV_BLOCK 4
#endif
#ifndef DINVK_TGV_TILE
#define DINVK_TGV_TILE 56
#endif
#ifndef DINVK_TGV_BLOCK
#define DINVK_TGV_BLOCK 2
#endif

#ifdef DINVK_EMUL
static inline void tv_fence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
template <typename T> static inline T tv_ldcg(const T* p) { return *p; }
#else
__device__ __forceinline__ void tv_fence() { __threadfence(); }
template <typename T> __device__ __forceinline__ T tv_ldcg(const T* p) { return __ldcg(p); }
#endif

namespace dinvk {
namespace tv {

// ---- stencils ------------------------------------------------------------------------------------------------------
// Each operator reads its field through an accessor f(dh, dw) = the field at (h + dh, w + dw); (h, w) is the image pixel,
// which the border tests need.

// p[c + dh * row + dw]: the accessor over a field stored row by row, in shared memory (I = int) or global memory (I = long long)
template <class P, class I>
struct Around {
  const P* p;
  I c;
  int row;
  __device__ __forceinline__ P operator()(int dh, int dw) const { return p[c + (I)dh * row + dw]; }
};
template <class P, class I>
__device__ __forceinline__ Around<P, I> around(const P* p, I c, int row) { return {p, c, row}; }

// nabla (tv.py:153-181): forward differences, zero on the last row / column
template <class X>
__device__ __forceinline__ float2 nabla(X x, int h, int w, int H, int W) {
  const float v = x(0, 0);
  return make_float2(h < H - 1 ? __fsub_rn(x(1, 0), v) : 0.f, w < W - 1 ? __fsub_rn(x(0, 1), v) : 0.f);
}

// nabla_adjoint in tv.py:202-216 order: vertical component first, then horizontal; each "-= own, += previous"
template <class G>
__device__ __forceinline__ float nabla_adjoint(G g, int h, int w, int H, int W) {
  float a = 0.f;
  if (h < H - 1) a = __fsub_rn(a, g(0, 0).x);
  if (h > 0) a = __fadd_rn(a, g(-1, 0).x);
  if (w < W - 1) a = __fsub_rn(a, g(0, 0).y);
  if (w > 0) a = __fadd_rn(a, g(0, -1).y);
  return a;
}

// TGVDenoiser.epsilon (tgv.py:229-270): (…,2) -> (…,4), component 2i + j = backward difference of field component i along
// axis j (0: H, 1: W), stored at the upper index; zero on the first row / column
template <class F>
__device__ __forceinline__ float4 epsilon(F f, int h, int w) {
  const float2 v = f(0, 0);
  float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
  if (h > 0) {
    const float2 a = f(-1, 0);
    e.x = __fsub_rn(v.x, a.x);
    e.z = __fsub_rn(v.y, a.y);
  }
  if (w > 0) {
    const float2 a = f(0, -1);
    e.y = __fsub_rn(v.x, a.x);
    e.w = __fsub_rn(v.y, a.y);
  }
  return e;
}

// TGVDenoiser.epsilon_adjoint (tgv.py:272-312): (…,4) -> (…,2), each component in the reference's order of updates
template <class G>
__device__ __forceinline__ float2 epsilon_adjoint(G g, int h, int w, int H, int W) {
  const float4 u = g(0, 0);
  float a0 = 0.f, a1 = 0.f;
  if (h < H - 1) {
    const float4 d = g(1, 0);
    a0 = __fsub_rn(a0, d.x);
    a1 = __fsub_rn(a1, d.z);
  }
  if (h > 0) {
    a0 = __fadd_rn(a0, u.x);
    a1 = __fadd_rn(a1, u.z);
  }
  if (w < W - 1) {
    const float4 e = g(0, 1);
    a0 = __fsub_rn(a0, e.y);
    a1 = __fsub_rn(a1, e.w);
  }
  if (w > 0) {
    a0 = __fadd_rn(a0, u.y);
    a1 = __fadd_rn(a1, u.w);
  }
  return make_float2(a0, a1);
}

// ---- the Chambolle-Pock scaffold -----------------------------------------------------------------------------------

// control block at the head of the workspace; zeroed by the first launch call of a prox
struct Ctrl {
  int ticket;    // CTAs of the current launch that have finished (the last one resets it)
  int it_done;   // iterations whose result is in state buffer `cur`
  int cur;       // 0/1: which ping-pong buffer holds the current state
  int status;    // RUNNING, FINISHED or REPLAY
  int replay_n;  // REPLAY: iterations to recompute from buffer `cur`
  int conv_j1;   // 1 + first converging sub-iteration of the converging launch, 0 if the break test never passed
  int pad[2];
};
enum { RUNNING = 0, FINISHED = 1, REPLAY = 2 };
constexpr size_t CTRL_BYTES = 64;

// what both CP kernels take besides their state buffers and per-sample constants
struct CpParams {
  Ctrl* ctrl;
  double* slots;  // (n_cta, 2K): per-CTA sums of the break test's numerator and denominator squares per sub-iteration
  int C, H, W, tiles_x, tiles_per_plane, n_cta, n_it_max;
  float crit, tau, one_plus_tau, sigma, rho;
};

// A CP kernel's tile: the T x T core a CTA owns, K iterations per launch, the region R x R staged around the core
// (HALO pixels on every side) and the region pixels per thread.
template <int T_, int K_, int HALO_>
struct Tile {
  static constexpr int T = T_, K = K_, HALO = HALO_, R = T + 2 * HALO, NT = 512, PPT = (R * R + NT - 1) / NT;
  static_assert(T >= 1 && K >= 1, "bad tile");
  static int tiles(int n) { return (n + T - 1) / T; }
  static __device__ __forceinline__ bool core(int r, int c) { return r >= HALO && r < HALO + T && c >= HALO && c < HALO + T; }
};

// This launch's place in the solve and this CTA's place in the image
struct Launch {
  bool replay;
  int it0, n, in, out;  // first iteration, iterations to run, ping-pong buffers read and written
  int plane, h0, w0;    // (b, c) plane, image pixel of the region's top-left corner
  long long off;        // the plane's offset in a (B, C, H, W) field
};

// Reads the control block; false: return now (the solve has finished or n_it_max is reached).  Every CTA reads the
// control block before any CTA of this launch can change it: only the last CTA to finish writes it.
template <class G>
__device__ __forceinline__ bool begin_launch(const CpParams& p, Launch& l) {
  const Ctrl* ctrl = p.ctrl;
  const int status = ctrl->status;
  if (status == FINISHED) return false;
  l.replay = status == REPLAY;
  l.it0 = ctrl->it_done;
  l.n = l.replay ? ctrl->replay_n : min(G::K, p.n_it_max - l.it0);
  l.in = ctrl->cur;
  l.out = l.in ^ 1;
  if (l.n <= 0) return false;
  l.plane = blockIdx.x / p.tiles_per_plane;
  const int tile = blockIdx.x % p.tiles_per_plane;
  l.h0 = (tile / p.tiles_x) * G::T - G::HALO;
  l.w0 = (tile % p.tiles_x) * G::T - G::HALO;
  l.off = (long long)l.plane * p.H * p.W;
  return true;
}

// buffer i of a ping-pong pair, at the plane's offset (no dynamic index into the parameter block)
template <class P>
__device__ __forceinline__ P* pick(P* const (&b)[2], int i, long long off) {
  return (i ? b[1] : b[0]) + off;
}

// f(i, idx, r, c, gh, gw) for each of this thread's region pixels (i-th of its PPT, region index idx = r R + c, image
// pixel (gh, gw)) whose region row and column lie in [lo, hi) and that lie inside the image.  Fully unrolled, so that
// per-pixel arrays indexed by i stay in registers.
template <class G, class F>
__device__ __forceinline__ void for_region(const Launch& l, int H, int W, int lo, int hi, F&& f) {
#pragma unroll
  for (int i = 0; i < G::PPT; ++i) {
    const int idx = threadIdx.x + i * G::NT;
    const int r = idx / G::R, c = idx % G::R;
    const int gh = l.h0 + r, gw = l.w0 + c;
    if (idx < G::R * G::R && r >= lo && r < hi && c >= lo && c < hi && gh >= 0 && gh < H && gw >= 0 && gw < W)
      f(i, idx, r, c, gh, gw);
  }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The end of a launch: this CTA's share of the break test goes to its own slot (no float atomics: the sums are
// reproducible run to run), and the last CTA to finish (atomic ticket) adds the slots in CTA order in fp64, applies the
// reference's test and writes the control block.  accd[s] sums (x_prev - x2)^2 and accn[s] the denominator's squares
// over the CTA's core after sub-iteration s.  EPS_OUTSIDE selects the denominator: TGV's ||x2|| + 1e-12 (tgv.py:162-164)
// rather than TV's ||x2 + 1e-12||, whose 1e-12 the caller has already added inside accn (tv.py:139-141).
template <class G, bool EPS_OUTSIDE>
__device__ __forceinline__ void finish_launch(const double (&accd)[G::K], const double (&accn)[G::K], const CpParams& p,
                                              const Launch& l) {
  constexpr int KB = G::K, NTB = G::NT, NWB = NTB / 32;
  __shared__ double red[NWB][2 * KB];
  __shared__ double tot[2 * KB];
  __shared__ int s_last;
  Ctrl* ctrl = p.ctrl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int s = 0; s < KB; ++s) {
    const double d = warp_sum(accd[s]), e = warp_sum(accn[s]);
    if (lane == 0) {
      red[warp][s] = d;
      red[warp][KB + s] = e;
    }
  }
  __syncthreads();
  if (tid < 2 * KB) {
    double v = 0.0;
    for (int w = 0; w < NWB; ++w) v += red[w][tid];
    p.slots[(long long)blockIdx.x * 2 * KB + tid] = v;
  }
  tv_fence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&ctrl->ticket, 1) == p.n_cta - 1;
  __syncthreads();
  if (!s_last) return;

  // last CTA: whole-tensor norms per sub-iteration, summed over the slots in CTA order in fp64
  tv_fence();
  for (int j = 0; j < 2 * KB; ++j) {
    double v = 0.0;
    for (int c = tid; c < p.n_cta; c += NTB) v += tv_ldcg(p.slots + (long long)c * 2 * KB + j);
    v = warp_sum(v);
    if (lane == 0) red[warp][0] = v;
    __syncthreads();
    if (tid == 0) {
      double t = 0.0;
      for (int w = 0; w < NWB; ++w) t += red[w][0];
      tot[j] = t;
    }
    __syncthreads();
  }
  if (tid == 0) {
    const int it0 = l.it0, n = l.n;
    if (l.replay) {
      ctrl->it_done = it0 + n;
      ctrl->cur = l.out;
      ctrl->status = FINISHED;
    } else {
      // the reference breaks after iteration it (0-based, counted in every call) when it > 1 and rel_err < crit, in fp32
      int j = -1;
      for (int s = 0; s < n; ++s) {
        if (it0 + s < 2) continue;
        const float num = (float)sqrt(tot[s]), den = (float)sqrt(tot[KB + s]);
        const float rel = num / (EPS_OUTSIDE ? __fadd_rn(den, 1e-12f) : den);
        if (rel < p.crit) { j = s; break; }
      }
      if (j < 0) {
        ctrl->it_done = it0 + n;
        ctrl->cur = l.out;
        ctrl->status = it0 + n >= p.n_it_max ? FINISHED : RUNNING;
      } else if (j == n - 1) {
        ctrl->it_done = it0 + n;
        ctrl->cur = l.out;
        ctrl->conv_j1 = j + 1;
        ctrl->status = FINISHED;
      } else {
        // converged inside the block: the next launch recomputes j + 1 iterations from this launch's (intact) input
        ctrl->replay_n = j + 1;
        ctrl->conv_j1 = j + 1;
        ctrl->status = REPLAY;
      }
    }
    ctrl->ticket = 0;
  }
}

// ---- TV prox -------------------------------------------------------------------------------------------------------

using TvTile = Tile<DINVK_TV_TILE, DINVK_TV_BLOCK, DINVK_TV_BLOCK>;
constexpr size_t TV_SMEM = sizeof(float) * 3 * TvTile::R * TvTile::R;  // v (R^2) + u2 (2 R^2)
static_assert(TvTile::R % 2 == 0, "u2 rows must stay 8-byte aligned");

struct TvParams {
  CpParams cp;
  const float* y;
  float* x2[2];
  float2* u2[2];
  const float* lambd;  // (B,)
  int mode;
};

// dual projection: mode 0 isotropic u / max(|u| / lambd, 1) (tv.py:75-82), mode 1 per-component clamp (tv.py:238-239).
// torch's clamp propagates NaN (fmaxf would not): lambd = 0 and u = 0 gives 0/0 = NaN exactly as the reference does.
__device__ __forceinline__ float2 dual_proj(float2 t, float l, int mode) {
  if (mode == 0) {
    const float n = sqrtf(__fmaf_rn(t.y, t.y, __fmul_rn(t.x, t.x)));  // torch's CPU vector_norm over two elements
    const float q = n / l;
    const float d = q != q ? q : fmaxf(q, 1.f);
    return make_float2(t.x / d, t.y / d);
  }
  const float ax = t.x != t.x ? t.x : fminf(fmaxf(t.x, -l), l);
  const float ay = t.y != t.y ? t.y : fminf(fmaxf(t.y, -l), l);
  return make_float2(ax, ay);
}

// y and x2 in the owning thread's registers; v = 2x - x2 and u2 (one float2 per pixel, the reference's (B,C,H,W,2)
// layout) in shared memory.  An iteration needs u2 one pixel up / left of x and v one pixel down / right of u.  Pixels
// outside the image are neither staged nor read: every stencil tests the image borders, as the reference's operators do.
__global__ void __launch_bounds__(TvTile::NT) tv_cp_kernel(TvParams p) {
  using G = TvTile;
  constexpr int R = G::R, K = G::K;
  Launch l;
  if (!begin_launch<G>(p.cp, l)) return;
  const int H = p.cp.H, W = p.cp.W;
  const float lam = p.lambd[l.plane / p.cp.C];
  const float tau = p.cp.tau, opt = p.cp.one_plus_tau, sigma = p.cp.sigma, rho = p.cp.rho;
  const float* __restrict__ yg = p.y + l.off;
  const float* __restrict__ xin = pick(p.x2, l.in, l.off);
  const float2* __restrict__ uin = pick(p.u2, l.in, l.off);

  DINVK_DYN_SMEM(float, sm);
  float* V = sm;                                     // v = 2x - x2 of the current iteration
  float2* U = reinterpret_cast<float2*>(sm + R * R);  // u2

  float yv[G::PPT], xv[G::PPT];
#pragma unroll
  for (int i = 0; i < G::PPT; ++i) yv[i] = xv[i] = 0.f;
  for_region<G>(l, H, W, 0, R, [&](int i, int idx, int, int, int gh, int gw) {
    const long long g = (long long)gh * W + gw;
    yv[i] = yg[g];
    xv[i] = xin[g];
    U[idx] = uin[g];
  });
  __syncthreads();

  double accd[K], accn[K];
#pragma unroll
  for (int s = 0; s < K; ++s) {
    accd[s] = 0.0;
    accn[s] = 0.0;
    if (s < l.n) {
      // x = prox_tau_fx(x2 - tau nabla_adjoint(u2), y); v = 2x - x2; x2 += rho (x - x2)   (tv.py:131-133, 135)
      // on [s + 1, R - s): reads u2 at [s, R - s)
      for_region<G>(l, H, W, s + 1, R - s, [&](int i, int idx, int r, int c, int gh, int gw) {
        const float a = nabla_adjoint(around(U, idx, R), gh, gw, H, W);
        const float xo = xv[i];
        const float xn = __fadd_rn(__fsub_rn(xo, __fmul_rn(tau, a)), __fmul_rn(tau, yv[i])) / opt;
        V[idx] = __fsub_rn(__fmul_rn(2.f, xn), xo);
        const float x2n = __fadd_rn(xo, __fmul_rn(rho, __fsub_rn(xn, xo)));
        xv[i] = x2n;
        if (G::core(r, c)) {
          const float d = __fsub_rn(xo, x2n), e = __fadd_rn(x2n, 1e-12f);
          accd[s] += (double)d * (double)d;
          accn[s] += (double)e * (double)e;
        }
      });
      __syncthreads();
      // u = prox_sigma_g_conj(u2 + sigma nabla(v), lambd); u2 += rho (u - u2)   (tv.py:134, 136)
      // on [s + 1, R - s - 1): reads v at [s + 1, R - s)
      for_region<G>(l, H, W, s + 1, R - s - 1, [&](int, int idx, int, int, int gh, int gw) {
        const float2 g = nabla(around(V, idx, R), gh, gw, H, W);
        const float2 uo = U[idx];
        const float2 t = make_float2(__fadd_rn(uo.x, __fmul_rn(sigma, g.x)), __fadd_rn(uo.y, __fmul_rn(sigma, g.y)));
        const float2 u = dual_proj(t, lam, p.mode);
        U[idx] = make_float2(__fadd_rn(uo.x, __fmul_rn(rho, __fsub_rn(u.x, uo.x))),
                             __fadd_rn(uo.y, __fmul_rn(rho, __fsub_rn(u.y, uo.y))));
      });
      __syncthreads();
    }
  }

  // write back the T x T core
  float* __restrict__ xout = pick(p.x2, l.out, l.off);
  float2* __restrict__ uout = pick(p.u2, l.out, l.off);
  for_region<G>(l, H, W, G::HALO, G::HALO + G::T, [&](int i, int idx, int, int, int gh, int gw) {
    const long long g = (long long)gh * W + gw;
    xout[g] = xv[i];
    uout[g] = U[idx];
  });
  // ||x_prev - x2|| / ||x2 + 1e-12|| < crit (tv.py:139-145)
  finish_launch<G, false>(accd, accn, p.cp, l);
}

// ---- TGV prox ------------------------------------------------------------------------------------------------------

using TgvTile = Tile<DINVK_TGV_TILE, DINVK_TGV_BLOCK, 2 * DINVK_TGV_BLOCK>;
constexpr size_t TGV_SMEM = sizeof(float) * 7 * TgvTile::R * TgvTile::R;  // u2 (4 R^2) + tmp / d (2 R^2) + v (R^2)

struct TgvParams {
  CpParams cp;
  const float* y;
  float* x2[2];
  float2* r2[2];
  float4* u2[2];
  const float* tl1;  // (B,) tau * lambda1
  const float* l2;   // (B,) lambda2
};

// t / max(|t|_2 / l, 1) with torch.maximum's NaN propagation (fmaxf would drop a NaN)
__device__ __forceinline__ float proj_den(float sq, float l) {
  const float q = sqrtf(sq) / l;
  return q != q ? q : fmaxf(q, 1.f);
}

// One iteration of tgv.py:149-160 reads, per output pixel, fields two stencils away:
//   tmp(q) = tau epsilon_adjoint(u2)(q)           reads u2 at q, q + e_h, q + e_w
//   x(p) = (x2 - nabla_adjoint(tmp) + tau y) / (1 + tau), r(p) = prox_tau_fr(r2 + tmp)   read tmp at p, p - e_h, p - e_w
//   d(q) = nabla(2x - x2)(q) - (2r - r2)(q)       reads v = 2x - x2 at q, q + e_h, q + e_w
//   u(p) = prox_sigma_g_conj(u2 + sigma epsilon(d))(p)   reads d at p, p - e_h, p - e_w
// so u2 stays valid on [2s, R - 2s) of the region after s iterations: with R = T + 4K the T x T core is valid after K.
// x2 and r2 stay valid one pixel wider, which never binds.  Per region pixel: y, x2, r2 and w = 2r - r2 in the owning
// thread's registers; u2 (one float4, the reference's (B,C,H,W,4) layout), tmp (float2, reused for d once x and r are
// done) and v in shared memory.  Four barriered passes per iteration: tmp; x, v, x2 and r, w, r2; d; u, u2.  Pixels
// outside the image are neither staged nor read: every stencil tests the image borders, as the reference's operators do
// (zero last row of nabla, zero first row of epsilon, the four-term adjoints).
__global__ void __launch_bounds__(TgvTile::NT) tgv_cp_kernel(TgvParams p) {
  using G = TgvTile;
  constexpr int R = G::R, K = G::K;
  Launch l;
  if (!begin_launch<G>(p.cp, l)) return;
  const int H = p.cp.H, W = p.cp.W;
  const float tl1 = p.tl1[l.plane / p.cp.C], l2 = p.l2[l.plane / p.cp.C];
  const float tau = p.cp.tau, opt = p.cp.one_plus_tau, sigma = p.cp.sigma, rho = p.cp.rho;
  const float* __restrict__ yg = p.y + l.off;
  const float* __restrict__ xin = pick(p.x2, l.in, l.off);
  const float2* __restrict__ rin = pick(p.r2, l.in, l.off);
  const float4* __restrict__ uin = pick(p.u2, l.in, l.off);

  DINVK_DYN_SMEM(float, sm);
  float4* U = reinterpret_cast<float4*>(sm);             // u2
  float2* D = reinterpret_cast<float2*>(sm + 4 * R * R);  // tmp, then d
  float* V = sm + 6 * R * R;                             // v = 2x - x2

  float yv[G::PPT], xv[G::PPT], r0[G::PPT], r1[G::PPT], w0v[G::PPT], w1v[G::PPT];
#pragma unroll
  for (int i = 0; i < G::PPT; ++i) yv[i] = xv[i] = r0[i] = r1[i] = w0v[i] = w1v[i] = 0.f;
  for_region<G>(l, H, W, 0, R, [&](int i, int idx, int, int, int gh, int gw) {
    const long long g = (long long)gh * W + gw;
    yv[i] = yg[g];
    xv[i] = xin[g];
    const float2 r = rin[g];
    r0[i] = r.x;
    r1[i] = r.y;
    U[idx] = uin[g];
  });
  __syncthreads();

  double accd[K], accn[K];
#pragma unroll
  for (int s = 0; s < K; ++s) {
    accd[s] = 0.0;
    accn[s] = 0.0;
    if (s < l.n) {
      // tmp = tau * epsilon_adjoint(u2) on [2s, R - 2s - 1)
      for_region<G>(l, H, W, 2 * s, R - 2 * s - 1, [&](int, int idx, int, int, int gh, int gw) {
        const float2 a = epsilon_adjoint(around(U, idx, R), gh, gw, H, W);
        D[idx] = make_float2(__fmul_rn(tau, a.x), __fmul_rn(tau, a.y));
      });
      __syncthreads();
      // x = prox_tau_fx(x2 - nabla_adjoint(tmp), y), v = 2x - x2, x2 += rho (x - x2);
      // r = prox_tau_fr(r2 + tmp, lambda1), w = 2r - r2, r2 += rho (r - r2)   on [2s + 1, R - 2s - 1)
      for_region<G>(l, H, W, 2 * s + 1, R - 2 * s - 1, [&](int i, int idx, int r, int c, int gh, int gw) {
        const float2 t = D[idx];
        const float a = nabla_adjoint(around(D, idx, R), gh, gw, H, W);
        const float xo = xv[i];
        const float xn = __fadd_rn(__fsub_rn(xo, a), __fmul_rn(tau, yv[i])) / opt;
        V[idx] = __fsub_rn(__fmul_rn(2.f, xn), xo);
        const float x2n = __fadd_rn(xo, __fmul_rn(rho, __fsub_rn(xn, xo)));
        xv[i] = x2n;
        if (G::core(r, c)) {
          const float d = __fsub_rn(xo, x2n);
          accd[s] += (double)d * (double)d;
          accn[s] += (double)x2n * (double)x2n;
        }
        // r - r / max(sqrt(s0^2 + s1^2) / (tau lambda1), 1), the last-axis sum left to right (tgv.py:76-83)
        const float s0 = __fadd_rn(r0[i], t.x), s1 = __fadd_rn(r1[i], t.y);
        const float m = proj_den(__fadd_rn(__fmul_rn(s0, s0), __fmul_rn(s1, s1)), tl1);
        const float q0 = __fsub_rn(s0, s0 / m), q1 = __fsub_rn(s1, s1 / m);
        w0v[i] = __fsub_rn(__fmul_rn(2.f, q0), r0[i]);
        w1v[i] = __fsub_rn(__fmul_rn(2.f, q1), r1[i]);
        r0[i] = __fadd_rn(r0[i], __fmul_rn(rho, __fsub_rn(q0, r0[i])));
        r1[i] = __fadd_rn(r1[i], __fmul_rn(rho, __fsub_rn(q1, r1[i])));
      });
      __syncthreads();
      // d = nabla(v) - w on [2s + 1, R - 2s - 2) (tmp is dead: d takes its place)
      for_region<G>(l, H, W, 2 * s + 1, R - 2 * s - 2, [&](int i, int idx, int, int, int gh, int gw) {
        const float2 g = nabla(around(V, idx, R), gh, gw, H, W);
        D[idx] = make_float2(__fsub_rn(g.x, w0v[i]), __fsub_rn(g.y, w1v[i]));
      });
      __syncthreads();
      // u = prox_sigma_g_conj(u2 + sigma epsilon(d), lambda2), u2 += rho (u - u2) on [2s + 2, R - 2s - 2)
      for_region<G>(l, H, W, 2 * s + 2, R - 2 * s - 2, [&](int, int idx, int, int, int gh, int gw) {
        const float4 e = epsilon(around(D, idx, R), gh, gw);
        const float4 uo = U[idx];
        const float t0 = __fadd_rn(uo.x, __fmul_rn(sigma, e.x)), t1 = __fadd_rn(uo.y, __fmul_rn(sigma, e.y));
        const float t2 = __fadd_rn(uo.z, __fmul_rn(sigma, e.z)), t3 = __fadd_rn(uo.w, __fmul_rn(sigma, e.w));
        const float sq = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(t0, t0), __fmul_rn(t1, t1)), __fmul_rn(t2, t2)), __fmul_rn(t3, t3));
        const float m = proj_den(sq, l2);
        U[idx] = make_float4(__fadd_rn(uo.x, __fmul_rn(rho, __fsub_rn(t0 / m, uo.x))),
                             __fadd_rn(uo.y, __fmul_rn(rho, __fsub_rn(t1 / m, uo.y))),
                             __fadd_rn(uo.z, __fmul_rn(rho, __fsub_rn(t2 / m, uo.z))),
                             __fadd_rn(uo.w, __fmul_rn(rho, __fsub_rn(t3 / m, uo.w))));
      });
      __syncthreads();
    }
  }

  // write back the T x T core
  float* __restrict__ xout = pick(p.x2, l.out, l.off);
  float2* __restrict__ rout = pick(p.r2, l.out, l.off);
  float4* __restrict__ uout = pick(p.u2, l.out, l.off);
  for_region<G>(l, H, W, G::HALO, G::HALO + G::T, [&](int i, int idx, int, int, int gh, int gw) {
    const long long g = (long long)gh * W + gw;
    xout[g] = xv[i];
    rout[g] = make_float2(r0[i], r1[i]);
    uout[g] = U[idx];
  });
  // ||x_prev - x2|| / (||x2|| + 1e-12) < crit (tgv.py:162-166)
  finish_launch<G, true>(accd, accn, p.cp, l);
}

// ---- host side of the CP proxes ------------------------------------------------------------------------------------

template <class G>
static size_t workspace_bytes(int B, int C, int H, int W) {
  const size_t n_cta = (size_t)std::max(B, 0) * std::max(C, 0) * G::tiles(std::max(H, 1)) * G::tiles(std::max(W, 1));
  return CTRL_BYTES + sizeof(double) * 2 * G::K * std::max<size_t>(n_cta, 1);
}

// What the two prox entry points share: checks the shape and the workspace, fills p.cp with the reference's constants
// (python doubles rounded once to fp32 by torch), clears the control block on the first call of a prox and issues
// n_launch launches of the kernel.
template <class G, class P>
static int run_cp(const char* name, void (*kernel)(P), size_t smem, P& p, int B, int C, int H, int W, int n_it_max, float crit,
                  double tau, double sigma, double rho, int first, int n_launch, void* workspace, size_t workspace_bytes,
                  void* stream) {
  DINVK_CHECK_ARG(B >= 0 && C >= 0 && H > 0 && W > 0 && n_it_max >= 0 && n_launch >= 0, "%s: bad shape", name);
  DINVK_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "%s: workspace must be 8-byte aligned", name);
  if (workspace_bytes < tv::workspace_bytes<G>(B, C, H, W)) return set_error(DINVK_EWORKSPACE, "%s: workspace too small", name);
  const long long n_cta = (long long)B * C * G::tiles(H) * G::tiles(W);
  DINVK_CHECK_ARG(n_cta < (1LL << 31), "%s: too many tiles", name);
  p.cp = CpParams{reinterpret_cast<Ctrl*>(workspace), reinterpret_cast<double*>(static_cast<char*>(workspace) + CTRL_BYTES), C, H, W,
                  G::tiles(W), G::tiles(H) * G::tiles(W), (int)n_cta, n_it_max, crit, (float)tau, (float)(1.0 + tau), (float)sigma,
                  (float)rho};
  if (first) {
    cudaError_t e = cudaMemsetAsync(workspace, 0, CTRL_BYTES, (cudaStream_t)stream);
    if (e != cudaSuccess) return set_error(DINVK_ECUDA, "%s: memset: %s", name, cudaGetErrorString(e));
  }
  if (n_cta == 0) return DINVK_OK;
  int rc;
#ifndef DINVK_EMUL
  // opt in even at exactly 48 KB of dynamic shared memory: the static reduction buffers come on top of it
  if ((rc = raise_smem_limit(reinterpret_cast<const void*>(kernel), smem))) return rc;
#endif
  for (int l = 0; l < n_launch; ++l) {
    DINVK_LAUNCH(kernel, dim3((unsigned)n_cta), dim3(G::NT), smem, stream, p);
    if ((rc = DINVK_POST_LAUNCH())) return rc;
  }
  return DINVK_OK;
}

// ---- stencil kernels -----------------------------------------------------------------------------------------------

// f(i, h, w) for every pixel i of a (planes, H, W) stack of n pixels, grid-stride
template <class F>
__device__ __forceinline__ void for_each_pixel(int H, int W, long long n, F&& f) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long plane = i / ((long long)H * W);
    const int hw = (int)(i - plane * H * W);
    f(i, hw / W, hw % W);
  }
}

__global__ void __launch_bounds__(256) nabla_kernel(const float* __restrict__ x, float2* __restrict__ g, int H, int W, long long n) {
  for_each_pixel(H, W, n, [&](long long i, int h, int w) { g[i] = nabla(around(x, i, W), h, w, H, W); });
}

__global__ void __launch_bounds__(256) nabla_adjoint_kernel(const float2* __restrict__ g, float* __restrict__ x, int H, int W, long long n) {
  for_each_pixel(H, W, n, [&](long long i, int h, int w) { x[i] = nabla_adjoint(around(g, i, W), h, w, H, W); });
}

__global__ void __launch_bounds__(256) epsilon_kernel(const float2* __restrict__ f, float4* __restrict__ g, int H, int W, long long n) {
  for_each_pixel(H, W, n, [&](long long i, int h, int w) { g[i] = epsilon(around(f, i, W), h, w); });
}

__global__ void __launch_bounds__(256) epsilon_adjoint_kernel(const float4* __restrict__ g, float2* __restrict__ f, int H, int W,
                                                              long long n) {
  for_each_pixel(H, W, n, [&](long long i, int h, int w) { f[i] = epsilon_adjoint(around(g, i, W), h, w, H, W); });
}

// TVPrior.grad (prior.py:544-572): nabla_adjoint(Dx / |Dx|), 0 where |Dx| = 0
__global__ void __launch_bounds__(256) tv_grad_kernel(const float* __restrict__ x, float* __restrict__ out, int H, int W, long long n) {
  for_each_pixel(H, W, n, [&](long long i, int h, int w) {
    out[i] = nabla_adjoint([&](int dh, int dw) {
      const float2 d = nabla(around(x, i + (long long)dh * W + dw, W), h + dh, w + dw, H, W);
      const float nrm = sqrtf(__fmaf_rn(d.y, d.y, __fmul_rn(d.x, d.x)));
      return nrm > 0.f ? make_float2(d.x / nrm, d.y / nrm) : make_float2(0.f, 0.f);
    }, h, w, H, W);
  });
}

__device__ __forceinline__ double block_sum(double v, double* part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) part[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r += part[w];
  __syncthreads();
  return r;  // valid in thread 0
}

// TVPrior.fn / TVL1Prior.fn (prior.py:507-522, 595-611), two deterministic stages like dinvk_batched_dot:
// partial[b, chunk] = sum over the chunk of |Dx| (mode 0: 2-norm over the two differences, mode 1: 1-norm)
__global__ void __launch_bounds__(256) tv_fn_partial_kernel(double* __restrict__ partial, const float* __restrict__ x, int mode,
                                                            int C, int H, int W, int chunks) {
  __shared__ double part[8];
  const int b = blockIdx.y, ch = blockIdx.x;
  const long long n_per = (long long)C * H * W;
  double acc = 0.0;
  for (long long i = (long long)ch * blockDim.x + threadIdx.x; i < n_per; i += (long long)chunks * blockDim.x) {
    const int c = (int)(i / ((long long)H * W));
    const int hw = (int)(i - (long long)c * H * W);
    const float2 d = nabla(around(x, (long long)b * n_per + i, W), hw / W, hw % W, H, W);
    acc += mode == 0 ? (double)sqrtf(__fadd_rn(__fmul_rn(d.x, d.x), __fmul_rn(d.y, d.y))) : (double)fabsf(d.x) + (double)fabsf(d.y);
  }
  const double r = block_sum(acc, part);
  if (threadIdx.x == 0) partial[(long long)b * chunks + ch] = r;
}

__global__ void __launch_bounds__(256) tv_fn_final_kernel(float* __restrict__ out, const double* __restrict__ partial, int chunks) {
  __shared__ double part[8];
  const int b = blockIdx.x;
  double acc = 0.0;
  for (int i = threadIdx.x; i < chunks; i += blockDim.x) acc += partial[(long long)b * chunks + i];
  const double r = block_sum(acc, part);
  if (threadIdx.x == 0) out[b] = (float)r;
}

static int stencil_grid(long long n) {
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  return (int)std::max(1LL, std::min(blocks, cap));
}

static int fn_chunks(int B, long long n_per) {
  long long want = (n_per + 256 * 16 - 1) / (256 * 16);
  const long long cap = std::max(1, sm_count() * 8 / std::max(1, B));
  return (int)std::max(1LL, std::min(want, cap));
}

}  // namespace tv
}  // namespace dinvk

using namespace dinvk;

extern "C" int dinvk_tv_block(int* tile, int* iters) {
  if (tile) *tile = tv::TvTile::T;
  if (iters) *iters = tv::TvTile::K;
  return DINVK_OK;
}

extern "C" size_t dinvk_tv_prox_workspace_bytes(int B, int C, int H, int W) { return tv::workspace_bytes<tv::TvTile>(B, C, H, W); }

extern "C" int dinvk_tv_prox(const float* y, float* x2_a, float* u2_a, float* x2_b, float* u2_b, const float* lambd, int B, int C,
                             int H, int W, int n_it_max, float crit, double tau, double rho, int mode, int first, int n_launch,
                             void* workspace, size_t workspace_bytes, void* stream) {
  DINVK_CHECK_ARG(y && x2_a && u2_a && x2_b && u2_b && lambd && workspace, "dinvk_tv_prox: null pointer");
  DINVK_CHECK_ARG(mode == 0 || mode == 1, "dinvk_tv_prox: mode must be 0 (TV) or 1 (TV-L1)");
  DINVK_CHECK_ARG((reinterpret_cast<uintptr_t>(u2_a) & 7) == 0 && (reinterpret_cast<uintptr_t>(u2_b) & 7) == 0,
                  "dinvk_tv_prox: u2 buffers must be 8-byte aligned");
  tv::TvParams p{{}, y, {x2_a, x2_b}, {reinterpret_cast<float2*>(u2_a), reinterpret_cast<float2*>(u2_b)}, lambd, mode};
  // sigma = 1 / tau / 2^(ndim - 1) with ndim = 4 (tv.py:119-121)
  return tv::run_cp<tv::TvTile>("dinvk_tv_prox", tv::tv_cp_kernel, tv::TV_SMEM, p, B, C, H, W, n_it_max, crit, tau, 1.0 / tau / 8.0,
                                rho, first, n_launch, workspace, workspace_bytes, stream);
}

extern "C" int dinvk_tv_stencil(int op, const float* in, float* out, int B, int C, int H, int W, void* stream) {
  DINVK_CHECK_ARG(in && out && B >= 0 && C >= 0 && H > 0 && W > 0, "dinvk_tv_stencil: bad arguments");
  DINVK_CHECK_ARG(op >= 0 && op <= 4,
                  "dinvk_tv_stencil: op must be 0 (nabla), 1 (nabla_adjoint), 2 (TV subgradient), 3 (epsilon) or 4 (epsilon_adjoint)");
  if (op >= 3)
    DINVK_CHECK_ARG((reinterpret_cast<uintptr_t>(in) & 7) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0 &&
                        (reinterpret_cast<uintptr_t>(op == 3 ? out : in) & 15) == 0,
                    "dinvk_tv_stencil: epsilon fields must be 8-byte (…,2) and 16-byte (…,4) aligned");
  const long long n = (long long)B * C * H * W;
  if (n == 0) return DINVK_OK;
  const dim3 grid(tv::stencil_grid(n));
  if (op == 0)
    DINVK_LAUNCH(tv::nabla_kernel, grid, dim3(256), 0, stream, in, reinterpret_cast<float2*>(out), H, W, n);
  else if (op == 1)
    DINVK_LAUNCH(tv::nabla_adjoint_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const float2*>(in), out, H, W, n);
  else if (op == 2)
    DINVK_LAUNCH(tv::tv_grad_kernel, grid, dim3(256), 0, stream, in, out, H, W, n);
  else if (op == 3)
    DINVK_LAUNCH(tv::epsilon_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const float2*>(in), reinterpret_cast<float4*>(out),
                 H, W, n);
  else
    DINVK_LAUNCH(tv::epsilon_adjoint_kernel, grid, dim3(256), 0, stream, reinterpret_cast<const float4*>(in),
                 reinterpret_cast<float2*>(out), H, W, n);
  return DINVK_POST_LAUNCH();
}

extern "C" int dinvk_tgv_block(int* tile, int* iters) {
  if (tile) *tile = tv::TgvTile::T;
  if (iters) *iters = tv::TgvTile::K;
  return DINVK_OK;
}

extern "C" size_t dinvk_tgv_prox_workspace_bytes(int B, int C, int H, int W) { return tv::workspace_bytes<tv::TgvTile>(B, C, H, W); }

extern "C" int dinvk_tgv_prox(const float* y, float* x2_a, float* r2_a, float* u2_a, float* x2_b, float* r2_b, float* u2_b,
                              const float* tl1, const float* l2, int B, int C, int H, int W, int n_it_max, float crit, double tau,
                              double rho, int first, int n_launch, void* workspace, size_t workspace_bytes, void* stream) {
  DINVK_CHECK_ARG(y && x2_a && r2_a && u2_a && x2_b && r2_b && u2_b && tl1 && l2 && workspace, "dinvk_tgv_prox: null pointer");
  DINVK_CHECK_ARG((reinterpret_cast<uintptr_t>(u2_a) & 15) == 0 && (reinterpret_cast<uintptr_t>(u2_b) & 15) == 0,
                  "dinvk_tgv_prox: u2 buffers must be 16-byte aligned");
  DINVK_CHECK_ARG((reinterpret_cast<uintptr_t>(r2_a) & 7) == 0 && (reinterpret_cast<uintptr_t>(r2_b) & 7) == 0,
                  "dinvk_tgv_prox: r2 buffers must be 8-byte aligned");
  tv::TgvParams p{{}, y, {x2_a, x2_b}, {reinterpret_cast<float2*>(r2_a), reinterpret_cast<float2*>(r2_b)},
                  {reinterpret_cast<float4*>(u2_a), reinterpret_cast<float4*>(u2_b)}, tl1, l2};
  // sigma = 1 / tau / 72 in 2-D (tgv.py:121-122)
  return tv::run_cp<tv::TgvTile>("dinvk_tgv_prox", tv::tgv_cp_kernel, tv::TGV_SMEM, p, B, C, H, W, n_it_max, crit, tau,
                                 1.0 / tau / 72.0, rho, first, n_launch, workspace, workspace_bytes, stream);
}

extern "C" size_t dinvk_tv_fn_workspace_bytes(int B, int C, int H, int W) {
  const long long n_per = (long long)std::max(C, 0) * std::max(H, 0) * std::max(W, 0);
  return sizeof(double) * (size_t)std::max(1, B) * (size_t)tv::fn_chunks(B, n_per) + 64;
}

extern "C" int dinvk_tv_fn(float* out, const float* x, int mode, int B, int C, int H, int W, void* workspace, size_t workspace_bytes,
                           void* stream) {
  DINVK_CHECK_ARG(out && x && workspace && B >= 0 && C >= 0 && H > 0 && W > 0, "dinvk_tv_fn: bad arguments");
  DINVK_CHECK_ARG(mode == 0 || mode == 1, "dinvk_tv_fn: mode must be 0 (TV) or 1 (TV-L1)");
  DINVK_CHECK_ARG(B <= 65535, "dinvk_tv_fn: batch too large");
  if (B == 0) return DINVK_OK;
  if (workspace_bytes < dinvk_tv_fn_workspace_bytes(B, C, H, W)) return set_error(DINVK_EWORKSPACE, "dinvk_tv_fn: workspace too small");
  const int chunks = tv::fn_chunks(B, (long long)C * H * W);
  double* partial = reinterpret_cast<double*>(((uintptr_t)workspace + 7) & ~(uintptr_t)7);
  DINVK_LAUNCH(tv::tv_fn_partial_kernel, dim3(chunks, B), dim3(256), 0, stream, partial, x, mode, C, H, W, chunks);
  DINVK_LAUNCH(tv::tv_fn_final_kernel, dim3(B), dim3(256), 0, stream, out, (const double*)partial, chunks);
  return DINVK_POST_LAUNCH();
}
