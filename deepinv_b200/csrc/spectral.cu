// spectral.cu — fused spectral ("decomposable") operator family: MRI and BlurFFT.
//
// Replaces the bodies of (reference, relative to the deepinv tree):
//   MRIMixin.to_torch_complex/from_torch_complex/fft/ifft   deepinv/utils/mixins.py:148-206
//   DecomposablePhysics.A/A_adjoint/A_adjoint_A/prox_l2/A_dagger  deepinv/physics/forward.py:1080-1252
//   MultiCoilMRI.A/A_adjoint                                 deepinv/physics/mri.py:254-324
//   BlurFFT.U/V/...                                          deepinv/physics/blur.py:639-692
//   L2.grad + fStepPGD (fused data step)                     deepinv/optim/data_fidelity.py:335-336, optim_iterators/pgd.py:137-139
//
// Data movement (DESIGN.md §3): a 2-D transform is two tile passes over HBM-resident images:
//   COL pass: one CTA owns a strip of Wc columns x all H rows of one image (coalesced Wc*4-byte
//             row segments), transforms along H in shared memory.
//   ROW pass: one CTA owns L full rows (fully contiguous), transforms along W; the mask / spectral
//             multiplier, and for A^T A / prox the inverse row transform, are fused into this pass.
// The intermediate between the two passes is an interleaved complex workspace written once and read
// once; for the cfg2 batch (33.5 MB) it stays resident in the 50 MB L2.  When the multiplier does
// not depend on h (Cartesian line masks, mask_sh == 0) and both transforms run, the H-direction
// transforms cancel algebraically and a single ROW pass does the whole operator.
#include "common.cuh"
#include "fft_core.cuh"

#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>
#include <vector>

namespace dinvk {

// ---------------------------------------------------------------------------------------------
// pass description
// ---------------------------------------------------------------------------------------------
struct PassParams {
  int B, H, W;          // B = number of complex images handled by this pass
  int wv;               // valid width of the planar global rows (== W except for zero-padded 1-D filtering)
  int lines;            // rows per CTA (ROW) or columns per CTA (COL)
  // source
  const float* p0; const float* p1; float a0, a1;
  int src_nc;           // planar source: number of coil planes interleaved per batch sample (>=1)
  int src_div;          // planar source batch index = image / src_div (coil broadcast of x)
  const float2* tin;    // interleaved source (B,H,W) if non-null
  const float2* coil;   // multiply source by coil map if non-null  (index by image/ncoil, image%ncoil)
  long long coil_sb; int ncoil;
  // transforms along this pass's axis
  int dir1, dir2;       // 0 none, -1 forward, +1 inverse
  int centered;         // centred transform (fast path computes the +-1 phases itself; the generic path uses pre/post)
  // pointwise multiplier
  int gmode; int g_at_load; int g_after;
  const float* g; long long gsb, gsc, gsh; float gc; const float* gcb;
  // destination
  float* out; int dst_nc; float2* tout;
  const float* q0; const float* q1; float e0, e1, e2;
  // tables for this axis
  const float2* tw; const float2* pre; const float2* post;
  FftPlanDev plan;
};

__device__ __forceinline__ float2 apply_g(const PassParams& P, float2 v, int img, int h, int w) {
  const int mb = img / P.ncoil;
  if (P.gmode == DINVK_G_CMUL || P.gmode == DINVK_G_CMUL_CONJ) {
    const float2 m = __ldg(reinterpret_cast<const float2*>(P.g) + (long long)mb * P.gsb + (long long)h * P.gsh + w);
    return P.gmode == DINVK_G_CMUL ? cmul(v, m) : cmul_conj(v, m);
  }
  const long long o = (long long)mb * P.gsb + (long long)h * P.gsh + w;
  float m0 = __ldg(P.g + o), m1 = __ldg(P.g + o + P.gsc);
  switch (P.gmode) {
    case DINVK_G_MASK: break;
    case DINVK_G_SQ: m0 = m0 * m0; m1 = m1 * m1; break;
    case DINVK_G_INV_SQ_PLUS_C: {
      const float c = P.gcb ? __ldg(P.gcb + mb) : P.gc;
      m0 = 1.0f / (m0 * m0 + c);
      m1 = 1.0f / (m1 * m1 + c);
      break;
    }
    case DINVK_G_PINV:
      m0 = m0 > 1e-5f ? 1.0f / m0 : 0.0f;
      m1 = m1 > 1e-5f ? 1.0f / m1 : 0.0f;
      break;
    default: break;
  }
  return make_float2(v.x * m0, v.y * m1);
}

// planar addressing of image `img` in a (batch, 2, nc, H, W) tensor: returns offset of the real plane,
// the imaginary plane is +cs
__device__ __forceinline__ long long planar_base(int img, int nc, long long HW, long long& cs) {
  cs = (long long)nc * HW;
  return (long long)(img / nc) * 2 * cs + (long long)(img % nc) * HW;
}

template <bool COLS, int NTHR>
__global__ void __launch_bounds__(NTHR, 1024 / NTHR) spectral_pass_kernel(const PassParams P) {
  DINVK_DYN_SMEM(float2, buf);
  const int tid = threadIdx.x;
  constexpr int nthr = NTHR;
  const int N = COLS ? P.H : P.W;          // transform length of this pass
  const long long HW = (long long)P.H * P.W;    // interleaved workspaces and coil maps
  const long long HWg = (long long)P.H * P.wv;  // planar global tensors

  // tile geometry
  int img0 = 0, c0 = 0;
  long long row0 = 0;
  int nlines = P.lines;
  if (COLS) {
    const int strips = (P.W + P.lines - 1) / P.lines;
    img0 = blockIdx.x / strips;
    c0 = (blockIdx.x % strips) * P.lines;
    nlines = min(P.lines, P.W - c0);
  } else {
    row0 = (long long)blockIdx.x * P.lines;
    const long long rows_total = (long long)P.B * P.H;
    nlines = (int)min((long long)P.lines, rows_total - row0);
  }
  RowLayout RL; RL.ls = row_line_stride(N);
  ColLayout CL; CL.lines = P.lines;
  const int telems = nlines * N;

  // ---- LOAD -----------------------------------------------------------------------------------
  for (int e = tid; e < telems; e += nthr) {
    int line, n, img, h, w;
    if (COLS) { n = e / nlines; line = e - n * nlines; img = img0; h = n; w = c0 + line; }
    else { line = e / N; n = e - line * N; const long long gr = row0 + line; img = (int)(gr / P.H); h = (int)(gr - (long long)img * P.H); w = n; }
    float2 v;
    if (P.tin) {
      v = P.tin[(long long)img * HW + (long long)h * P.W + w];
    } else {
      long long cs;
      const long long o = planar_base(img / P.src_div, P.src_nc, HWg, cs) + (long long)h * P.wv + w;
      if (w < P.wv) {
        v = make_float2(P.a0 * __ldg(P.p0 + o), P.a0 * __ldg(P.p0 + o + cs));
        if (P.p1) { v.x += P.a1 * __ldg(P.p1 + o); v.y += P.a1 * __ldg(P.p1 + o + cs); }
      } else {
        v = make_float2(0.f, 0.f);
      }
    }
    if (P.coil) {
      const float2 s = __ldg(P.coil + (long long)(img / P.ncoil) * P.coil_sb + (long long)(img % P.ncoil) * HW + (long long)h * P.W + w);
      v = cmul(v, s);
    }
    if (P.g_at_load) v = apply_g(P, v, img, h, w);
    if (P.dir1 != 0) {
      if (P.dir1 > 0) v = cconj(v);
      v = cmul(v, __ldg(P.pre + n));
    }
    buf[COLS ? CL.idx(line, n) : RL.idx(line, n)] = v;
  }
  __syncthreads();

  // ---- transform 1 ----------------------------------------------------------------------------
  if (P.dir1 != 0) {
    if (COLS) fft_tile(buf, P.tw, P.plan, P.lines, tid, nthr, CL);
    else fft_tile(buf, P.tw, P.plan, nlines, tid, nthr, RL);
  }

  // ---- fused middle: post-phase of transform 1, multiplier, pre-phase of transform 2 ----------
  if (P.dir2 != 0) {
    for (int e = tid; e < telems; e += nthr) {
      int line, n, img, h, w;
      if (COLS) { n = e / nlines; line = e - n * nlines; img = img0; h = n; w = c0 + line; }
      else { line = e / N; n = e - line * N; const long long gr = row0 + line; img = (int)(gr / P.H); h = (int)(gr - (long long)img * P.H); w = n; }
      const int si = COLS ? CL.idx(line, n) : RL.idx(line, n);
      float2 v = buf[si];
      if (P.dir1 != 0) { v = cmul(v, __ldg(P.post + n)); if (P.dir1 > 0) v = cconj(v); }
      if (P.g_after) v = apply_g(P, v, img, h, w);
      if (P.dir2 > 0) v = cconj(v);
      v = cmul(v, __ldg(P.pre + n));
      buf[si] = v;
    }
    __syncthreads();
    if (COLS) fft_tile(buf, P.tw, P.plan, P.lines, tid, nthr, CL);
    else fft_tile(buf, P.tw, P.plan, nlines, tid, nthr, RL);
  }

  // ---- STORE ----------------------------------------------------------------------------------
  const int last_dir = P.dir2 != 0 ? P.dir2 : P.dir1;
  for (int e = tid; e < telems; e += nthr) {
    int line, n, img, h, w;
    if (COLS) { n = e / nlines; line = e - n * nlines; img = img0; h = n; w = c0 + line; }
    else { line = e / N; n = e - line * N; const long long gr = row0 + line; img = (int)(gr / P.H); h = (int)(gr - (long long)img * P.H); w = n; }
    float2 v = buf[COLS ? CL.idx(line, n) : RL.idx(line, n)];
    if (last_dir != 0) { v = cmul(v, __ldg(P.post + n)); if (last_dir > 0) v = cconj(v); }
    if (P.dir2 == 0 && P.g_after) v = apply_g(P, v, img, h, w);
    if (P.tout) {
      P.tout[(long long)img * HW + (long long)h * P.W + w] = v;
    } else if (w < P.wv) {
      long long cs;
      const long long o = planar_base(img, P.dst_nc, HWg, cs) + (long long)h * P.wv + w;
      float re = P.e0 * v.x, im = P.e0 * v.y;
      if (P.q0) { re += P.e1 * __ldg(P.q0 + o); im += P.e1 * __ldg(P.q0 + o + cs); }
      if (P.q1) { re += P.e2 * __ldg(P.q1 + o); im += P.e2 * __ldg(P.q1 + o + cs); }
      P.out[o] = re;
      P.out[o + cs] = im;
    }
  }
}

}  // namespace dinvk
#include "spectral_fast.cuh"
#include "spectral_pipe.cuh"
#include "spectral_pipe320.cuh"
namespace dinvk {

// O(N^2) DFT along one axis of an interleaved (B,H,W) tensor — sizes with prime factors > 5.
// out[k] = N^-1/2 * sum_n in[n] * w^{(k-c)(n-c)}  (c = N/2 when centred, else 0); dir = -1 fwd / +1 inv
__global__ void dft_axis_naive_kernel(const float2* __restrict__ in, float2* __restrict__ out, int B, int H, int W,
                                      int axis_w, int dir, int centered, const float2* __restrict__ tw) {
  const long long total = (long long)B * H * W;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid < total) {
    const int w = (int)(gid % W);
    const int h = (int)((gid / W) % H);
    const long long img = gid / ((long long)W * H);
    const int N = axis_w ? W : H;
    const int k = axis_w ? w : h;
    const int c = centered ? N / 2 : 0;
    const long long base = img * (long long)H * W + (axis_w ? (long long)h * W : w);
    const long long stride = axis_w ? 1 : W;
    float2 acc = make_float2(0.f, 0.f);
    long long kk = ((long long)(k - c) % N + N) % N;
    for (int n = 0; n < N; ++n) {
      const long long nn = ((long long)(n - c) % N + N) % N;
      const int ti = (int)((kk * nn) % N);
      float2 t = __ldg(tw + ti);
      if (dir > 0) t.y = -t.y;
      const float2 x = in[base + n * stride];
      acc.x += x.x * t.x - x.y * t.y;
      acc.y += x.x * t.y + x.y * t.x;
    }
    const float sc = 1.0f / sqrtf((float)N);
    out[gid] = make_float2(acc.x * sc, acc.y * sc);
  }
}

// coil combination after the per-coil inverse transforms (deepinv/physics/mri.py:313-322):
// mode 2: out[b] = sum_n conj(S[b,n]) * v[b,n]   (planar (batch,2,H,W))
// mode 3: out[b] = sqrt(sum_n |v[b,n]|^2)        ((batch,1,H,W))
__global__ void coil_combine_kernel(const float2* __restrict__ v, const float2* __restrict__ S, long long coil_sb,
                                    float* __restrict__ out, int batch, int ncoil, long long HW, int mode, float e0) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid < (long long)batch * HW) {
    const long long b = gid / HW, p = gid - b * HW;
    float re = 0.f, im = 0.f;
    for (int n = 0; n < ncoil; ++n) {
      const float2 x = v[(b * ncoil + n) * HW + p];
      if (mode == 2) {
        const float2 s = __ldg(S + b * coil_sb + (long long)n * HW + p);
        re += x.x * s.x + x.y * s.y;
        im += x.y * s.x - x.x * s.y;
      } else {
        re += x.x * x.x + x.y * x.y;
      }
    }
    if (mode == 2) { out[b * 2 * HW + p] = e0 * re; out[b * 2 * HW + HW + p] = e0 * im; }
    else out[b * HW + p] = sqrtf(re);
  }
}

// ---------------------------------------------------------------------------------------------
// host side: table cache
// ---------------------------------------------------------------------------------------------
struct Tables { float2* tw; float2* pre; float2* post; };

static void unit_root(long long num, long long den, double* c, double* s) {
  // exp(2*pi*i*num/den) with exact values on the axes
  num %= den; if (num < 0) num += den;
  if ((4 * num) % den == 0) {
    const long long q = 4 * num / den;
    const double cc[4] = {1, 0, -1, 0}, ss[4] = {0, 1, 0, -1};
    *c = cc[q]; *s = ss[q];
    return;
  }
  const double a = 2.0 * 3.14159265358979323846264338327950288 * (double)num / (double)den;
  *c = cos(a); *s = sin(a);
}

static std::mutex g_tab_mu;
static std::map<std::vector<int>, Tables> g_tab;

static int get_tables(int n, int centered, Tables* out) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_tab_mu);
  std::vector<int> key = {dev, n, centered};
  auto it = g_tab.find(key);
  if (it != g_tab.end()) { *out = it->second; return 0; }
  std::vector<float2> tw(n), pre(n), post(n);
  const long long c = centered ? n / 2 : 0;
  const double sc = 1.0 / sqrt((double)n);
  for (int k = 0; k < n; ++k) {
    double cr, ci;
    unit_root(-(long long)k, n, &cr, &ci);
    tw[k] = make_float2((float)cr, (float)ci);
    unit_root(c * k, n, &cr, &ci);                     // exp(+2*pi*i*c*n/N)
    pre[k] = make_float2((float)cr, (float)ci);
    unit_root(c * k - c * c, n, &cr, &ci);             // exp(+2*pi*i*c*k/N - 2*pi*i*c^2/N) / sqrt(N)
    post[k] = make_float2((float)(cr * sc), (float)(ci * sc));
  }
  Tables t;
  float2* base = nullptr;
  if (cudaMalloc((void**)&base, sizeof(float2) * 3 * (size_t)n) != cudaSuccess)
    return set_error(DINVK_ECUDA, "cudaMalloc of FFT tables (n=%d) failed", n);
  t.tw = base; t.pre = base + n; t.post = base + 2 * (size_t)n;
  cudaMemcpy(t.tw, tw.data(), sizeof(float2) * n, cudaMemcpyHostToDevice);
  cudaMemcpy(t.pre, pre.data(), sizeof(float2) * n, cudaMemcpyHostToDevice);
  cudaMemcpy(t.post, post.data(), sizeof(float2) * n, cudaMemcpyHostToDevice);
  g_tab[key] = t;
  *out = t;
  return 0;
}


static inline bool al16(const void* p);
#ifdef DINVK_EMUL
template <typename K, typename... Args>
static void launch_pdl(K kern, unsigned grid, unsigned block, size_t smem, void* stream, const Args&... args) {
  (void)stream;
  count_launch();
  ::emul::launch(dim3(grid), dim3(block), smem, [&]() { kern(args...); });
}
#else
// launch with programmatic stream serialization (PDL): the kernel may begin its prologue while the previous kernel in the
// stream drains; it executes griddepcontrol.wait before touching memory (see spectral_pipe.cuh)
template <typename K, typename... Args>
static void launch_pdl(K kern, unsigned grid, unsigned block, size_t smem, void* stream, const Args&... args) {
  count_launch();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = getenv("DINVK_NO_PDL") ? 0 : 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  (void)cudaLaunchKernelEx(&cfg, kern, args...);
}
#endif
// 256x256 single-coil fast path (spectral_pipe.cuh).  Returns -1 when the call does not qualify.
static int try_pipe(const dinvk_spectral_args& a, float2* T1, const Tables& tW, void* stream) {
  if (a.H != 256 || a.W != 256 || a.ncoil > 1) return -1;
  if (getenv("DINVK_NO_PIPE_FFT")) return -1;
  if (!(a.fwd || a.inv)) return -1;
  if (a.gmode == DINVK_G_CMUL || a.gmode == DINVK_G_CMUL_CONJ) return -1;
  if (!al16(a.p0) || !al16(a.p1) || !al16(a.q0) || !al16(a.q1) || !al16(a.out) || !al16(a.mask)) return -1;
  if (a.gmode != DINVK_G_NONE && ((a.mask_sb & 1) || (a.mask_sc & 1) || (a.mask_sh & 1))) return -1;
  const bool fused = a.fwd && a.inv;
  if (fused && a.gmode != DINVK_G_NONE && (a.mask_sh != 0 || a.mask_sc != 0)) return -1;  // full masks: 3 tile passes
  sp::PipeParams P = sp::PipeParams();
  P.B = a.B;
  P.p0 = a.p0; P.p1 = a.p1; P.a0 = a.a0; P.a1 = a.p1 ? a.a1 : 0.f;
  P.gmode = a.gmode; P.g = a.mask; P.gsb = a.mask_sb; P.gsc = a.mask_sc; P.gsh = a.mask_sh; P.gc = a.c; P.gcb = a.c_batch;
  P.q0 = a.q0; P.q1 = a.q1; P.e0 = a.e0; P.e1 = a.q0 ? a.e1 : 0.f; P.e2 = a.q1 ? a.e2 : 0.f;
  P.out = a.out; P.ws = T1; P.tw = tW.tw; P.centered = a.centered ? 1 : 0;
  const int ntiles = a.B * 16;
  static const int occ = getenv("DINVK_SP_OCC3") ? 3 : 2;  // CTAs per SM of the row kernels (3 = 24 warps at <= 85 registers: measured no faster)
  const unsigned grid = (unsigned)std::min(ntiles, occ * sm_count());
  const unsigned grid2 = (unsigned)std::min(ntiles, 2 * sm_count());
  int rc;
#define DINVK_SP_LAUNCH(KERN)                                                        \
  do {                                                                               \
    if (occ == 2) {                                                                  \
      if ((rc = allow_smem(KERN<true, 2>, sp::ROW_SMEM))) return rc;                 \
      if ((rc = allow_smem(KERN<false, 2>, sp::ROW_SMEM))) return rc;                \
      if (a.p1) launch_pdl(KERN<true, 2>, grid, sp::NT, sp::ROW_SMEM, stream, P);    \
      else launch_pdl(KERN<false, 2>, grid, sp::NT, sp::ROW_SMEM, stream, P);        \
    } else {                                                                         \
      if ((rc = allow_smem(KERN<true, 3>, sp::ROW_SMEM))) return rc;                 \
      if ((rc = allow_smem(KERN<false, 3>, sp::ROW_SMEM))) return rc;                \
      if (a.p1) launch_pdl(KERN<true, 3>, grid, sp::NT, sp::ROW_SMEM, stream, P);    \
      else launch_pdl(KERN<false, 3>, grid, sp::NT, sp::ROW_SMEM, stream, P);        \
    }                                                                                \
  } while (0)
  if (fused) {
    DINVK_SP_LAUNCH(sp::sp_row_fused);
    return DINVK_POST_LAUNCH();
  }
  P.inverse = a.inv ? 1 : 0;
  P.g_at_load = a.inv ? 1 : 0;  // A^T: multiplier on the k-space source; A: multiplier on the k-space result
  DINVK_SP_LAUNCH(sp::sp_pass1);
#undef DINVK_SP_LAUNCH
  if ((rc = DINVK_POST_LAUNCH())) return rc;
  if ((rc = allow_smem(sp::sp_pass2, sp::P2_SMEM))) return rc;
  launch_pdl(sp::sp_pass2, grid2, sp::P2_NT, sp::P2_SMEM, stream, P);
  return DINVK_POST_LAUNCH();
}
// 320x320 two-pass path (spectral_pipe320.cuh): A and A^T, single- or multi-coil.  Returns -1 when the call does not qualify.
// `coil_ws` != null: pass 2 writes interleaved per-coil images there (the caller runs the coil reduction afterwards).
static int try_pipe320(const dinvk_spectral_args& a, float2* T1, float2* coil_ws, const Tables& tW, void* stream) {
  if (a.H != 320 || a.W != 320) return -1;
  if (getenv("DINVK_NO_PIPE_FFT")) return -1;
  if (a.fwd == a.inv) return -1;  // fused forward-inverse passes stay on the tile passes
  if (a.gmode == DINVK_G_CMUL || a.gmode == DINVK_G_CMUL_CONJ) return -1;
  if (!al16(a.p0) || !al16(a.p1) || !al16(a.out) || !al16(a.coil_maps)) return -1;
  const int nc = a.ncoil > 1 ? a.ncoil : 1;
  sp320::Params P = sp320::Params();
  P.B = a.B;
  P.p0 = a.p0; P.p1 = a.p1; P.a0 = a.a0; P.a1 = a.p1 ? a.a1 : 0.f;
  P.src_nc = 1; P.src_div = 1; P.ncoil = nc; P.dst_nc = 1;
  if (nc > 1 && a.coil_mode == 1) { P.src_div = nc; P.coil = reinterpret_cast<const float2*>(a.coil_maps); P.coil_sb = a.coil_sb; P.dst_nc = nc; }
  else if (nc > 1) { P.src_nc = nc; }
  P.gmode = a.gmode; P.g = a.mask; P.gsb = a.mask_sb; P.gsc = a.mask_sc; P.gsh = a.mask_sh; P.gc = a.c; P.gcb = a.c_batch;
  P.q0 = a.q0; P.q1 = a.q1; P.e0 = a.e0; P.e1 = a.q0 ? a.e1 : 0.f; P.e2 = a.q1 ? a.e2 : 0.f;
  P.out = a.out; P.tout = coil_ws; P.ws = T1; P.tw = tW.tw; P.centered = a.centered ? 1 : 0;
  P.inverse = a.inv ? 1 : 0;
  P.g_at_load = a.inv ? 1 : 0;
  if (coil_ws) { P.e0 = 1.f; P.q0 = nullptr; P.q1 = nullptr; P.e1 = 0.f; P.e2 = 0.f; }  // e0 is applied by the coil reduction
  int rc;
  if ((rc = allow_smem(sp320::sp320_pass1<true>, sp320::P1_SMEM))) return rc;
  if ((rc = allow_smem(sp320::sp320_pass1<false>, sp320::P1_SMEM))) return rc;
  if ((rc = allow_smem(sp320::sp320_pass2, sp320::P2_SMEM))) return rc;
  // one launch pair for the whole batch.  (Chunks of 64 images, whose 52 MB intermediate would stay in L2, measured
  // 10 % SLOWER at cfg4 — 210 vs 191 us: the passes are bound by issue / shared-memory exchange, not by the intermediate's
  // HBM round trip, and every extra launch pays a pipeline ramp.  `img0` keeps the chunked form available.)
  const int CH = 1 << 30;
  for (int i0 = 0; i0 < a.B; i0 += CH) {
    P.img0 = i0;
    P.B = std::min(CH, a.B - i0);
    const unsigned g1 = (unsigned)std::min(P.B * sp320::HB, 2 * sm_count());
    const unsigned g2 = (unsigned)std::min(P.B * sp320::HA, 2 * sm_count());
    if (a.p1) launch_pdl(sp320::sp320_pass1<true>, g1, sp320::NT, sp320::P1_SMEM, stream, P);
    else launch_pdl(sp320::sp320_pass1<false>, g1, sp320::NT, sp320::P1_SMEM, stream, P);
    launch_pdl(sp320::sp320_pass2, g2, sp320::NT, sp320::P2_SMEM, stream, P);
  }
  return DINVK_POST_LAUNCH();
}


static int pow2floor(int x) { int p = 1; while (2 * p <= x) p *= 2; return p; }

struct TileCfg { int lines; int nthr; size_t smem; };

// tiles hold at most 16 complex elements per thread (15 when a radix-3/5 stage is present: a thread
// owns floor(16/R) butterflies, see stage_load)
static int tile_budget(const FftPlan& p, int nthr) {
  for (int s = 0; s < p.nstages; ++s)
    if (p.radix[s] == 3 || p.radix[s] == 5) return 15 * nthr;
  return 16 * nthr;
}
static bool row_cfg(const FftPlan& pW, int W, TileCfg* c) {
  int nthr = 256;
  while ((long long)W > tile_budget(pW, nthr) && nthr < 1024) nthr *= 2;
  if ((long long)W > tile_budget(pW, nthr)) return false;
  int lines = tile_budget(pW, nthr) / W;
  if (lines < 1) lines = 1;
  if (lines > 64) lines = 64;
  c->lines = lines; c->nthr = nthr;
  c->smem = (size_t)lines * row_line_stride(W) * sizeof(float2);
  return true;
}
static bool col_cfg(const FftPlan& pH, int H, int W, TileCfg* c) {
  // prefer 16-column strips (64-byte row segments x 2 planes); never narrower than 4 columns
  int nthr = 256;
  while ((long long)H * 16 > tile_budget(pH, nthr) && nthr < 1024) nthr *= 2;
  int wc = pow2floor((int)std::min<long long>(16, std::max(1, tile_budget(pH, nthr) / H)));
  if ((long long)wc * H > tile_budget(pH, nthr)) return false;
  if (wc < 4 && wc < W) return false;
  if (wc > W) wc = W;
  c->lines = wc; c->nthr = nthr;
  c->smem = (size_t)wc * H * sizeof(float2);
  return true;
}

template <bool COLS, int NTHR>
static int launch_pass_t(PassParams& P, const TileCfg& cfg, void* stream) {
  int rc;
  if ((rc = allow_smem(spectral_pass_kernel<COLS, NTHR>, cfg.smem))) return rc;
  unsigned grid;
  if (COLS) grid = (unsigned)P.B * (unsigned)ceil_div(P.W, cfg.lines);
  else grid = (unsigned)ceil_div((long long)P.B * P.H, cfg.lines);
  auto kern = spectral_pass_kernel<COLS, NTHR>;
  DINVK_LAUNCH(kern, dim3(grid), dim3(NTHR), cfg.smem, stream, P);
  return DINVK_POST_LAUNCH();
}
static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int LOGN, bool COLS, int NTHR, int LINES>
static int launch_fast_t(PassParams& P, void* stream) {
  constexpr int N = 1 << LOGN;
  const size_t smem = COLS ? (size_t)16 * N * sizeof(float2) : (size_t)LINES * (N + (N >> 4) + 1) * sizeof(float2);
  auto kern = spectral_fast_kernel<LOGN, COLS, NTHR, LINES>;
  int rc;
  if ((rc = allow_smem(kern, smem))) return rc;
  const unsigned grid = COLS ? (unsigned)P.B * (unsigned)(P.W >> 4) : (unsigned)P.B * (unsigned)(P.H / LINES);
  P.lines = LINES;
  DINVK_LAUNCH(kern, dim3(grid), dim3(NTHR), smem, stream, P);
  return DINVK_POST_LAUNCH();
}

// power-of-two fast path; returns -1 when the pass does not qualify (caller falls back to the generic kernel)
static int try_launch_fast(bool cols, PassParams& P, void* stream) {
  static const bool disabled = getenv("DINVK_NO_FAST_FFT") != nullptr;
  if (disabled) return -1;
  const int N = cols ? P.H : P.W;
  if (N < 64 || N > 1024 || (N & (N - 1))) return -1;
  if (P.wv != P.W || (P.W & 3)) return -1;
  if (!al16(P.p0) || !al16(P.p1) || !al16(P.q0) || !al16(P.q1) || !al16(P.out) || !al16(P.tin) || !al16(P.tout) || !al16(P.coil) || !al16(P.g)) return -1;
  if (P.gmode != DINVK_G_NONE && ((P.gsb & 3) || (P.gsc & 3) || (P.gsh & 3))) return -1;
  if (P.gmode == DINVK_G_CMUL || P.gmode == DINVK_G_CMUL_CONJ) { if ((P.gsb & 1) || (P.gsh & 1)) return -1; }
  if (((long long)P.H * P.W) & 3) return -1;
  if (cols) {
    if (P.W & 15) return -1;
    switch (N) {
      case 128: return launch_fast_t<7, true, 128, 16>(P, stream);
      case 256: return launch_fast_t<8, true, 256, 16>(P, stream);
      case 512: return launch_fast_t<9, true, 512, 16>(P, stream);
      case 1024: return launch_fast_t<10, true, 1024, 16>(P, stream);
      default: return -1;
    }
  }
  const int lines = 4096 / N;
  if (P.H % lines) return -1;
  switch (N) {
    case 64: return launch_fast_t<6, false, 256, 64>(P, stream);
    case 128: return launch_fast_t<7, false, 256, 32>(P, stream);
    case 256: return launch_fast_t<8, false, 256, 16>(P, stream);
    case 512: return launch_fast_t<9, false, 256, 8>(P, stream);
    case 1024: return launch_fast_t<10, false, 256, 4>(P, stream);
    default: return -1;
  }
}

static int launch_pass(bool cols, PassParams& P, const TileCfg& cfg, void* stream) {
  if (P.dir1 != 0) {
    const int rc = try_launch_fast(cols, P, stream);
    if (rc >= 0) return rc;
  }
  P.lines = cfg.lines;
  if (cols) {
    switch (cfg.nthr) {
      case 256: return launch_pass_t<true, 256>(P, cfg, stream);
      case 512: return launch_pass_t<true, 512>(P, cfg, stream);
      default: return launch_pass_t<true, 1024>(P, cfg, stream);
    }
  }
  switch (cfg.nthr) {
    case 256: return launch_pass_t<false, 256>(P, cfg, stream);
    case 512: return launch_pass_t<false, 512>(P, cfg, stream);
    default: return launch_pass_t<false, 1024>(P, cfg, stream);
  }
}

static void init_pass(PassParams& P, const dinvk_spectral_args& a) {
  P = PassParams();
  P.B = a.B; P.H = a.H; P.W = a.W; P.wv = a.W; P.centered = a.centered ? 1 : 0;
  P.src_nc = 1; P.src_div = 1; P.dst_nc = 1; P.ncoil = a.ncoil > 1 ? a.ncoil : 1;
  P.a0 = 1.f; P.a1 = 0.f; P.e0 = 1.f; P.e1 = 0.f; P.e2 = 0.f;
  P.gmode = DINVK_G_NONE;
}
static void set_source(PassParams& P, const dinvk_spectral_args& a) {
  P.p0 = a.p0; P.p1 = a.p1; P.a0 = a.a0; P.a1 = a.p1 ? a.a1 : 0.f;
  if (a.ncoil > 1 && a.coil_mode == 1) {  // x (batch,2,H,W) broadcast over coils and multiplied by the maps
    P.src_nc = 1; P.src_div = a.ncoil;
    P.coil = reinterpret_cast<const float2*>(a.coil_maps); P.coil_sb = a.coil_sb;
  } else if (a.ncoil > 1) {               // y (batch,2,ncoil,H,W)
    P.src_nc = a.ncoil; P.src_div = 1;
  }
}
static void set_mult(PassParams& P, const dinvk_spectral_args& a, bool at_load) {
  P.gmode = a.gmode;
  if (a.gmode == DINVK_G_NONE) return;
  P.g = a.mask; P.gsb = a.mask_sb; P.gsc = a.mask_sc; P.gsh = a.mask_sh; P.gc = a.c; P.gcb = a.c_batch;
  P.g_at_load = at_load ? 1 : 0; P.g_after = at_load ? 0 : 1;
}
// destination = user output with epilogue, or the interleaved workspace when a coil reduction follows
static void set_dest(PassParams& P, const dinvk_spectral_args& a, float2* coil_ws) {
  if (coil_ws) { P.tout = coil_ws; return; }
  P.out = a.out; P.q0 = a.q0; P.q1 = a.q1; P.e0 = a.e0; P.e1 = a.q0 ? a.e1 : 0.f; P.e2 = a.q1 ? a.e2 : 0.f;
  P.dst_nc = (a.ncoil > 1 && a.coil_mode == 1) ? a.ncoil : 1;
}
static void set_axis(PassParams& P, const Tables& t, const FftPlan& plan) { P.tw = t.tw; P.pre = t.pre; P.post = t.post; P.plan = pack_plan(plan); }

}  // namespace dinvk

using namespace dinvk;

extern "C" size_t dinvk_spectral_workspace_bytes(int B, int H, int W) {
  return 2 * (size_t)B * (size_t)H * (size_t)W * sizeof(float2) + 256;
}

extern "C" int dinvk_fft_prepare(int n, int centered) {
  DINVK_CHECK_ARG(n >= 1, "dinvk_fft_prepare: n=%d", n);
  Tables t;
  return get_tables(n, centered ? 1 : 0, &t);
}

extern "C" int dinvk_spectral(const dinvk_spectral_args* ap, void* workspace, size_t workspace_bytes, void* stream) {
  DINVK_CHECK_ARG(ap != nullptr, "dinvk_spectral: null args");
  const dinvk_spectral_args& a = *ap;
  DINVK_CHECK_ARG(a.B >= 0 && a.H >= 1 && a.W >= 1, "dinvk_spectral: bad shape B=%d H=%d W=%d", a.B, a.H, a.W);
  DINVK_CHECK_ARG(a.p0 && a.out, "dinvk_spectral: p0/out must not be null");
  DINVK_CHECK_ARG(a.gmode >= DINVK_G_NONE && a.gmode <= DINVK_G_CMUL_CONJ, "dinvk_spectral: bad gmode %d", a.gmode);
  DINVK_CHECK_ARG(a.gmode == DINVK_G_NONE || a.mask, "dinvk_spectral: gmode %d needs a mask", a.gmode);
  const int nc = a.ncoil > 1 ? a.ncoil : 1;
  if (nc > 1) {
    DINVK_CHECK_ARG(a.coil_mode >= 1 && a.coil_mode <= 3, "dinvk_spectral: ncoil=%d needs coil_mode 1..3", nc);
    DINVK_CHECK_ARG(a.B % nc == 0, "dinvk_spectral: B=%d not a multiple of ncoil=%d", a.B, nc);
    DINVK_CHECK_ARG(a.coil_mode == 3 || a.coil_maps, "dinvk_spectral: coil maps missing");
    DINVK_CHECK_ARG(!(a.coil_mode == 1) || (a.fwd && !a.inv), "dinvk_spectral: coil_mode 1 is the forward operator");
    DINVK_CHECK_ARG(!(a.coil_mode >= 2) || (!a.fwd && a.inv), "dinvk_spectral: coil_mode 2/3 is the adjoint operator");
    DINVK_CHECK_ARG(!(a.coil_mode >= 2) || (!a.q0 && !a.q1), "dinvk_spectral: epilogue terms unsupported with coil reduction");
  }
  if (a.B == 0) return DINVK_OK;
  const size_t need = dinvk_spectral_workspace_bytes(a.B, a.H, a.W);
  DINVK_CHECK_ARG(workspace != nullptr || (!a.fwd && !a.inv), "dinvk_spectral: workspace is null");
  if (workspace_bytes < need && (a.fwd || a.inv)) return set_error(DINVK_EWORKSPACE, "dinvk_spectral: workspace %zu < %zu", workspace_bytes, need);
  const long long HW = (long long)a.H * a.W;
  uintptr_t wsp = ((uintptr_t)workspace + 127) & ~(uintptr_t)127;
  float2* T1 = reinterpret_cast<float2*>(wsp);
  float2* T2 = T1 + (size_t)a.B * HW;
  const bool coil_reduce = nc > 1 && a.coil_mode >= 2;

  Tables tH, tW;
  FftPlan pH = FftPlan(), pW = FftPlan();
  int rc;
  const int cen = a.centered ? 1 : 0;
  if ((rc = get_tables(a.H, cen, &tH))) return rc;
  if ((rc = get_tables(a.W, cen, &tW))) return rc;
  TileCfg rcfg, ccfg;
  const bool okH = make_fft_plan(a.H, &pH), okW = make_fft_plan(a.W, &pW);  // both always initialised
  const bool fast = okH && okW && row_cfg(pW, a.W, &rcfg) && col_cfg(pH, a.H, a.W, &ccfg);
  PassParams P;

  if (!a.fwd && !a.inv) {  // pure elementwise
    TileCfg ecfg; ecfg.nthr = 256; ecfg.lines = std::max(1, 4096 / a.W); ecfg.smem = (size_t)ecfg.lines * row_line_stride(a.W) * sizeof(float2);
    init_pass(P, a); set_source(P, a); set_mult(P, a, true); set_dest(P, a, nullptr);
    set_axis(P, tW, pW);
    return launch_pass(false, P, ecfg, stream);
  }

  if (fast) {
    const int prc = try_pipe(a, T1, tW, stream);
    if (prc >= 0) return prc;
  }
  if (fast) {
    if (a.fwd && !a.inv) {
      const int prc = try_pipe320(a, T1, nullptr, tW, stream);
      if (prc >= 0) return prc;
    }
    if (a.fwd && !a.inv) {
      // A: COL(fwd) planar -> T1 ; ROW(fwd, multiplier) T1 -> out
      init_pass(P, a); set_source(P, a); P.dir1 = -1; P.tout = T1; set_axis(P, tH, pH);
      if ((rc = launch_pass(true, P, ccfg, stream))) return rc;
      init_pass(P, a); P.tin = T1; P.dir1 = -1; set_mult(P, a, false); set_dest(P, a, nullptr); set_axis(P, tW, pW);
      return launch_pass(false, P, rcfg, stream);
    }
    int prc320 = -1;
    if (!a.fwd && a.inv) {
      prc320 = try_pipe320(a, T1, coil_reduce ? T2 : nullptr, tW, stream);
      if (prc320 > 0) return prc320;
    }
    if (!a.fwd && a.inv && prc320 == 0) {
      // done by the 320 x 320 two-pass kernels; a coil reduction (below) may follow
    } else if (!a.fwd && a.inv) {
      // A^T: ROW(multiplier at load, inv) planar -> T1 ; COL(inv) T1 -> out (or coil workspace)
      init_pass(P, a); set_source(P, a); set_mult(P, a, true); P.dir1 = +1; P.tout = T1; set_axis(P, tW, pW);
      if ((rc = launch_pass(false, P, rcfg, stream))) return rc;
      init_pass(P, a); P.tin = T1; P.dir1 = +1; set_dest(P, a, coil_reduce ? T2 : nullptr); set_axis(P, tH, pH);
      if ((rc = launch_pass(true, P, ccfg, stream))) return rc;
    } else {
      const bool complex_mult = a.gmode == DINVK_G_CMUL || a.gmode == DINVK_G_CMUL_CONJ;
      if (a.gmode == DINVK_G_NONE || (a.mask_sh == 0 && (complex_mult || a.mask_sc == 0))) {
        // multiplier independent of h and acting as a complex scalar (same factor on the real and
        // imaginary planes): it commutes with the H-direction transform, F_H^-1 F_H cancels
        // -> one fused ROW pass
        init_pass(P, a); set_source(P, a); P.dir1 = -1; P.dir2 = +1; set_mult(P, a, false); set_dest(P, a, nullptr); set_axis(P, tW, pW);
        return launch_pass(false, P, rcfg, stream);
      }
      init_pass(P, a); set_source(P, a); P.dir1 = -1; P.tout = T1; set_axis(P, tH, pH);
      if ((rc = launch_pass(true, P, ccfg, stream))) return rc;
      init_pass(P, a); P.tin = T1; P.dir1 = -1; P.dir2 = +1; set_mult(P, a, false); P.tout = T2; set_axis(P, tW, pW);
      if ((rc = launch_pass(false, P, rcfg, stream))) return rc;
      init_pass(P, a); P.tin = T2; P.dir1 = +1; set_dest(P, a, nullptr); set_axis(P, tH, pH);
      return launch_pass(true, P, ccfg, stream);
    }
  } else {
    // generic sizes: elementwise prologue -> naive axis DFTs -> elementwise epilogue
    TileCfg ecfg; ecfg.nthr = 256; ecfg.lines = std::max(1, 4096 / a.W); ecfg.smem = (size_t)ecfg.lines * row_line_stride(a.W) * sizeof(float2);
    const long long total = (long long)a.B * HW;
    const dim3 ngrid((unsigned)ceil_div(total, 256));
    float2 *cur = T1, *oth = T2;
    init_pass(P, a); set_source(P, a); if (!a.fwd) set_mult(P, a, true); P.tout = cur; set_axis(P, tW, pW);
    if ((rc = launch_pass(false, P, ecfg, stream))) return rc;
    if (a.fwd) {
      DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, cur, oth, a.B, a.H, a.W, 0, -1, cen, tH.tw);
      DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, oth, cur, a.B, a.H, a.W, 1, -1, cen, tW.tw);
      if ((rc = DINVK_POST_LAUNCH())) return rc;
      if (a.inv) {  // multiplier in the middle
        init_pass(P, a); P.tin = cur; set_mult(P, a, true); P.tout = oth; set_axis(P, tW, pW);
        if ((rc = launch_pass(false, P, ecfg, stream))) return rc;
        float2* t = cur; cur = oth; oth = t;
      }
    }
    if (a.inv) {
      DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, cur, oth, a.B, a.H, a.W, 1, +1, cen, tW.tw);
      DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, oth, cur, a.B, a.H, a.W, 0, +1, cen, tH.tw);
      if ((rc = DINVK_POST_LAUNCH())) return rc;
    }
    if (coil_reduce) {
      if (cur != T2) { cudaMemcpyAsync(T2, cur, sizeof(float2) * (size_t)total, cudaMemcpyDeviceToDevice, (cudaStream_t)stream); }
    } else {
      init_pass(P, a); P.tin = cur; if (a.fwd && !a.inv) set_mult(P, a, true); set_dest(P, a, nullptr); set_axis(P, tW, pW);
      return launch_pass(false, P, ecfg, stream);
    }
  }
  if (coil_reduce) {
    const int batch = a.B / nc;
    DINVK_LAUNCH(coil_combine_kernel, dim3((unsigned)ceil_div((long long)batch * HW, 256)), dim3(256), 0, stream,
                 (const float2*)T2, reinterpret_cast<const float2*>(a.coil_maps), (long long)a.coil_sb, a.out, batch, nc, HW,
                 a.coil_mode, a.e0);
    return DINVK_POST_LAUNCH();
  }
  return DINVK_OK;
}

// ---------------------------------------------------------------------------------------------
// 3-D: the same contract on contiguous (D,H,W) volumes.  Every axis is a pass of the 2-D family over its own view of the
// same memory, so the 3-D operator issues no copy and no permute:
//   depth  COL pass over one (D, H*W) "image" per volume: a CTA owns a strip of consecutive (h,w) columns and all D planes,
//          so its global accesses are the column pass's coalesced row segments; the coil maps (batch|1, ncoil, D, H, W) are
//          (ncoil, D, H*W) images in this view, which is where the forward operator multiplies by them;
//   H      COL pass over the B*D slices (H, W) of the interleaved workspace;
//   W      ROW pass over one (D*H, W) "image" per volume: the planar (batch,2,ncoil,D,H,W) layout and the multiplier
//          mask[b*sb + ch*sc + (d*H + h)*sh + w] are the 2-D addressing with D*H rows, so the mask is applied here.
// ---------------------------------------------------------------------------------------------
extern "C" size_t dinvk_spectral3d_workspace_bytes(int B, int D, int H, int W) {
  return 2 * (size_t)B * (size_t)D * (size_t)H * (size_t)W * sizeof(float2) + 256;
}

extern "C" int dinvk_spectral3d(const dinvk_spectral_args* ap, int D, void* workspace, size_t workspace_bytes, void* stream) {
  DINVK_CHECK_ARG(ap != nullptr, "dinvk_spectral3d: null args");
  const dinvk_spectral_args& a = *ap;
  DINVK_CHECK_ARG(a.B >= 0 && D >= 1 && a.H >= 1 && a.W >= 1, "dinvk_spectral3d: bad shape B=%d D=%d H=%d W=%d", a.B, D, a.H, a.W);
  const long long vol = (long long)D * a.H * a.W;
  DINVK_CHECK_ARG(vol < (1LL << 31), "dinvk_spectral3d: a volume of D*H*W = %lld elements (D=%d H=%d W=%d) exceeds 2^31 - 1", vol, D,
                  a.H, a.W);
  DINVK_CHECK_ARG((long long)a.B * D < (1LL << 31), "dinvk_spectral3d: B*D = %lld slices exceeds 2^31 - 1", (long long)a.B * D);
  DINVK_CHECK_ARG(a.p0 && a.out, "dinvk_spectral3d: p0/out must not be null");
  DINVK_CHECK_ARG(a.gmode >= DINVK_G_NONE && a.gmode <= DINVK_G_CMUL_CONJ, "dinvk_spectral3d: bad gmode %d", a.gmode);
  DINVK_CHECK_ARG(a.gmode == DINVK_G_NONE || a.mask, "dinvk_spectral3d: gmode %d needs a mask", a.gmode);
  const bool coils = a.coil_mode != 0;
  const int nc = coils ? a.ncoil : std::max(a.ncoil, 1);  // coil_mode 0: ncoil planar volumes per sample, no maps
  if (coils) {
    DINVK_CHECK_ARG(a.coil_mode >= 1 && a.coil_mode <= 3, "dinvk_spectral3d: bad coil_mode %d", a.coil_mode);
    DINVK_CHECK_ARG(nc >= 1, "dinvk_spectral3d: coil_mode %d needs ncoil >= 1, got %d", a.coil_mode, nc);
    DINVK_CHECK_ARG(a.B % nc == 0, "dinvk_spectral3d: B=%d not a multiple of ncoil=%d", a.B, nc);
    DINVK_CHECK_ARG(a.coil_mode == 3 || a.coil_maps, "dinvk_spectral3d: coil maps missing");
    DINVK_CHECK_ARG(!(a.coil_mode == 1) || (a.fwd && !a.inv), "dinvk_spectral3d: coil_mode 1 is the forward operator");
    DINVK_CHECK_ARG(!(a.coil_mode >= 2) || (!a.fwd && a.inv), "dinvk_spectral3d: coil_mode 2/3 is the adjoint operator");
    DINVK_CHECK_ARG(!(a.coil_mode >= 2) || (!a.q0 && !a.q1), "dinvk_spectral3d: epilogue terms unsupported with coil reduction");
  } else {
    DINVK_CHECK_ARG(a.B % nc == 0, "dinvk_spectral3d: B=%d not a multiple of ncoil=%d", a.B, nc);
  }
  if (a.B == 0) return DINVK_OK;
  const size_t need = dinvk_spectral3d_workspace_bytes(a.B, D, a.H, a.W);
  DINVK_CHECK_ARG(workspace != nullptr || (!a.fwd && !a.inv), "dinvk_spectral3d: workspace is null");
  if (workspace_bytes < need && (a.fwd || a.inv)) return set_error(DINVK_EWORKSPACE, "dinvk_spectral3d: workspace %zu < %zu", workspace_bytes, need);
  const int HW = a.H * a.W;
  uintptr_t wsp = ((uintptr_t)workspace + 127) & ~(uintptr_t)127;
  float2* T1 = reinterpret_cast<float2*>(wsp);
  float2* T2 = T1 + (size_t)a.B * vol;
  const bool coil_reduce = coils && a.coil_mode >= 2;

  Tables tD, tH, tW;
  FftPlan pD = FftPlan(), pH = FftPlan(), pW = FftPlan();
  int rc;
  const int cen = a.centered ? 1 : 0;
  if ((rc = get_tables(D, cen, &tD))) return rc;
  if ((rc = get_tables(a.H, cen, &tH))) return rc;
  if ((rc = get_tables(a.W, cen, &tW))) return rc;
  TileCfg dcfg, hcfg, wcfg;
  const bool okD = make_fft_plan(D, &pD), okH = make_fft_plan(a.H, &pH), okW = make_fft_plan(a.W, &pW);  // all initialised
  // an axis runs as a tile pass when its plan and tile fit; the fused paths below need all three
  const bool tileD = okD && col_cfg(pD, D, HW, &dcfg);
  const bool tileH = okH && col_cfg(pH, a.H, a.W, &hcfg);
  const bool tileW = okW && row_cfg(pW, a.W, &wcfg);
  const bool fast = tileD && tileH && tileW;

  // pass parameters on one of the three views; the source / destination are the user's planar tensors or a workspace
  PassParams P;
  auto depth = [&]() { init_pass(P, a); P.B = a.B; P.H = D; P.W = HW; P.wv = HW; set_axis(P, tD, pD); };
  auto slice = [&]() { init_pass(P, a); P.B = a.B * D; P.H = a.H; P.W = a.W; P.wv = a.W; set_axis(P, tH, pH); };
  auto rows = [&]() { init_pass(P, a); P.B = a.B; P.H = D * a.H; P.W = a.W; P.wv = a.W; set_axis(P, tW, pW); };
  auto source = [&]() {
    P.p0 = a.p0; P.p1 = a.p1; P.a0 = a.a0; P.a1 = a.p1 ? a.a1 : 0.f;
    if (a.coil_mode == 1) { P.src_div = nc; P.coil = reinterpret_cast<const float2*>(a.coil_maps); P.coil_sb = a.coil_sb; }
    else P.src_nc = nc;
  };
  auto dest = [&](float2* ws) {
    if (ws) { P.tout = ws; return; }
    P.out = a.out; P.q0 = a.q0; P.q1 = a.q1; P.e0 = a.e0; P.e1 = a.q0 ? a.e1 : 0.f; P.e2 = a.q1 ? a.e2 : 0.f;
    P.dst_nc = a.coil_mode <= 1 ? nc : 1;
  };
  TileCfg ecfg; ecfg.nthr = 256; ecfg.lines = std::max(1, 4096 / a.W); ecfg.smem = (size_t)ecfg.lines * row_line_stride(a.W) * sizeof(float2);

  if (!a.fwd && !a.inv) {  // pure elementwise
    rows(); source(); set_mult(P, a, true); dest(nullptr);
    return launch_pass(false, P, ecfg, stream);
  }
  float2* red = nullptr;  // interleaved per-coil volumes for the coil reduction
  if (fast) {
    if (a.fwd && !a.inv) {
      // A: depth(fwd, coil maps) planar -> T1 ; H(fwd) T1 -> T2 ; W(fwd, multiplier) T2 -> out
      depth(); source(); P.dir1 = -1; P.tout = T1;
      if ((rc = launch_pass(true, P, dcfg, stream))) return rc;
      slice(); P.tin = T1; P.dir1 = -1; P.tout = T2;
      if ((rc = launch_pass(true, P, hcfg, stream))) return rc;
      rows(); P.tin = T2; P.dir1 = -1; set_mult(P, a, false); dest(nullptr);
      return launch_pass(false, P, wcfg, stream);
    }
    if (!a.fwd && a.inv) {
      // A^T: W(multiplier at load, inv) planar -> T1 ; H(inv) T1 -> T2 ; depth(inv) T2 -> out (or T1 for the coil reduction)
      rows(); source(); set_mult(P, a, true); P.dir1 = +1; P.tout = T1;
      if ((rc = launch_pass(false, P, wcfg, stream))) return rc;
      slice(); P.tin = T1; P.dir1 = +1; P.tout = T2;
      if ((rc = launch_pass(true, P, hcfg, stream))) return rc;
      red = coil_reduce ? T1 : nullptr;
      depth(); P.tin = T2; P.dir1 = +1; dest(red);
      if ((rc = launch_pass(true, P, dcfg, stream))) return rc;
    } else {
      // A^T A / prox / data step: depth, H, W(fwd, multiplier, inv), H, depth(epilogue)
      depth(); source(); P.dir1 = -1; P.tout = T1;
      if ((rc = launch_pass(true, P, dcfg, stream))) return rc;
      slice(); P.tin = T1; P.dir1 = -1; P.tout = T2;
      if ((rc = launch_pass(true, P, hcfg, stream))) return rc;
      rows(); P.tin = T2; P.dir1 = -1; P.dir2 = +1; set_mult(P, a, false); P.tout = T1;
      if ((rc = launch_pass(false, P, wcfg, stream))) return rc;
      slice(); P.tin = T1; P.dir1 = +1; P.tout = T2;
      if ((rc = launch_pass(true, P, hcfg, stream))) return rc;
      depth(); P.tin = T2; P.dir1 = +1; dest(nullptr);
      return launch_pass(true, P, dcfg, stream);
    }
  } else {
    // an axis with a prime factor above 5 (or beyond the tile budget): elementwise prologue -> one transform per axis on the
    // interleaved workspace (a tile pass where the axis allows one, else the O(N^2) DFT) -> elementwise epilogue (or the
    // coil reduction)
    const long long total = (long long)a.B * vol;
    const dim3 ngrid((unsigned)ceil_div(total, 256));
    float2 *cur = T1, *oth = T2;
    auto axis = [&](int ax, int dir) -> int {  // ax 0 depth, 1 H, 2 W
      const bool tile = ax == 0 ? tileD : ax == 1 ? tileH : tileW;
      int r = 0;
      if (tile) {
        if (ax == 0) depth(); else if (ax == 1) slice(); else rows();
        P.tin = cur; P.tout = oth; P.dir1 = dir;
        r = launch_pass(ax != 2, P, ax == 0 ? dcfg : ax == 1 ? hcfg : wcfg, stream);
      } else if (ax == 0) {
        DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, cur, oth, a.B, D, HW, 0, dir, cen, tD.tw);
      } else {
        DINVK_LAUNCH(dft_axis_naive_kernel, ngrid, dim3(256), 0, stream, cur, oth, a.B * D, a.H, a.W, ax == 2 ? 1 : 0, dir, cen,
                     ax == 2 ? tW.tw : tH.tw);
      }
      std::swap(cur, oth);
      return r;
    };
    rows(); source(); if (!a.fwd) set_mult(P, a, true); P.tout = cur;
    if ((rc = launch_pass(false, P, ecfg, stream))) return rc;
    if (a.fwd) {
      for (int ax = 0; ax < 3; ++ax)
        if ((rc = axis(ax, -1))) return rc;
      if ((rc = DINVK_POST_LAUNCH())) return rc;
      if (a.inv) {  // multiplier in the middle
        rows(); P.tin = cur; set_mult(P, a, true); P.tout = oth;
        if ((rc = launch_pass(false, P, ecfg, stream))) return rc;
        std::swap(cur, oth);
      }
    }
    if (a.inv) {
      for (int ax = 2; ax >= 0; --ax)
        if ((rc = axis(ax, +1))) return rc;
      if ((rc = DINVK_POST_LAUNCH())) return rc;
    }
    if (coil_reduce) {
      red = cur;
    } else {
      rows(); P.tin = cur; if (a.fwd && !a.inv) set_mult(P, a, true); dest(nullptr);
      return launch_pass(false, P, ecfg, stream);
    }
  }
  if (!red) return DINVK_OK;
  // coil reduction: out[b] = e0 sum_n conj(S[b,n]) v[b,n] (coil_mode 2) or sqrt(sum_n |v[b,n]|^2) (coil_mode 3)
  const int batch = a.B / nc;
  DINVK_LAUNCH(coil_combine_kernel, dim3((unsigned)ceil_div((long long)batch * vol, 256)), dim3(256), 0, stream,
               (const float2*)red, reinterpret_cast<const float2*>(a.coil_maps), (long long)a.coil_sb, a.out, batch, nc, vol,
               a.coil_mode, a.e0);
  return DINVK_POST_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// ramp filter (FBP): rows of length N zero-padded to L, multiplied by 2*rfft(f) in the Fourier domain.
// Two real rows are packed as one complex signal (the filter is real and even, so real and imaginary
// parts filter independently); the ROW pass runs load(+pad) -> FFT -> multiply -> iFFT -> store(crop).
// ---------------------------------------------------------------------------------------------
namespace dinvk {
static std::mutex g_ramp_mu;
static std::map<std::vector<int>, float*> g_ramp;

static int ramp_padded_len(int N) {
  int L = 64;
  while (L < 2 * N) L *= 2;  // max(64, 2^ceil(log2(2N)))  (radon.py:96-98)
  return L;
}
static int get_ramp_table(int L, float** out) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_ramp_mu);
  std::vector<int> key = {dev, L};
  auto it = g_ramp.find(key);
  if (it != g_ramp.end()) { *out = it->second; return 0; }
  // f[0] = 1/4, f[odd k] = -1/(pi n)^2 with n = 1,3,..,L/2-1,L/2-1,..,3,1  (radon.py:151-162); f is even,
  // so its DFT is real: F[k] = sum_n f[n] cos(2 pi k n / L); the multiplier is 2 F, stored for all L bins.
  std::vector<double> f(L, 0.0);
  f[0] = 0.25;
  {
    std::vector<double> nn;
    for (int v = 1; v < L / 2 + 1; v += 2) nn.push_back(v);
    for (int v = L / 2 - 1; v > 0; v -= 2) nn.push_back(v);
    size_t q = 0;
    for (int k = 1; k < L; k += 2) { const double d = 3.14159265358979323846264338327950288 * nn[q++]; f[k] = -1.0 / (d * d); }
  }
  std::vector<float> mult(L);
  for (int k = 0; k <= L / 2; ++k) {
    double acc = 0.0;
    for (int n = 0; n < L; ++n) {
      double c, s;
      unit_root((long long)k * n, L, &c, &s);
      acc += f[n] * c;
    }
    mult[k] = (float)(2.0 * acc);
    if (k > 0 && k < L - k) mult[L - k] = mult[k];
  }
  float* d = nullptr;
  if (cudaMalloc((void**)&d, sizeof(float) * (size_t)L) != cudaSuccess) return set_error(DINVK_ECUDA, "cudaMalloc of ramp table failed");
  cudaMemcpy(d, mult.data(), sizeof(float) * (size_t)L, cudaMemcpyHostToDevice);
  g_ramp[key] = d;
  *out = d;
  return 0;
}
}  // namespace dinvk

namespace dinvk {
// Accuracy of the FFT-based filter: the rounding noise of an fp32 transform is proportional to the norm of its INPUT, and a
// sinogram row is dominated by its mean, which the ramp filter (all but) annihilates — the filtered row is ~100x smaller than
// the row, so the noise floor sits at ~5e-6 of the result (the reference's torch.fft path has the same property: 3.7e-6 on a
// 512 x 512 test image, and back-projection amplifies it to 2e-5).  The filter is linear: with m the row mean and box the
// indicator of the N valid samples,  filter(x) = filter(x - m box) + m filter(box);  filter(box) = B is a fixed vector per N,
// built once in double.  The transform then only sees the small residual x - m.
__global__ void __launch_bounds__(256) ramp_mean_sub_kernel(const float* __restrict__ x, float* __restrict__ xc, float* __restrict__ means,
                                                            int N) {
  __shared__ double part[8];
  const long long row = blockIdx.x;
  const float* src = x + row * N;
  double acc = 0.0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) acc += (double)__ldg(src + i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  double tot = 0.0;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += part[w];
  const float m = (float)(tot / (double)N);
  if (threadIdx.x == 0) means[row] = m;
  float* dst = xc + row * N;
  for (int i = threadIdx.x; i < N; i += blockDim.x) dst[i] = __ldg(src + i) - m;
}
__global__ void __launch_bounds__(256) ramp_add_box_kernel(float* __restrict__ out, const float* __restrict__ means,
                                                           const float* __restrict__ boxresp, int N) {
  const long long row = blockIdx.x;
  const float m = __ldg(means + row);
  float* dst = out + row * N;
  for (int i = threadIdx.x; i < N; i += blockDim.x) dst[i] = fmaf(m, __ldg(boxresp + i), dst[i]);
}
// EXACT spatial form of the same filter.  Zero-padding to L >= 2N makes the circular convolution a linear one on the N valid
// samples, and the reference's spatial kernel (radon.py:151-162) has the closed form g[0] = 1/2, g[d] = 0 for even d,
// g[d] = -2 / (pi d)^2 for odd d:   out[n] = x[n] / 2 - (2 / pi^2) sum_{m: n-m odd} x[m] / (n - m)^2.
// The sum is a difference of large terms (a sinogram row is ~100x larger than its filtered version), so it is accumulated in
// fp64: one CTA per row, the row split by parity into two double arrays in shared memory (an output of one parity only reads
// samples of the other), thread = output, lanes = consecutive outputs of one parity -> consecutive 8-byte reads.
// N^2 / 2 DFMA per row: 1.5 G for a 32 x 180 x 725 sinogram.  Result: the filter to fp32 rounding (1e-7) instead of the 4e-6 of
// an fp32 FFT — and FBP closer to its exact value than the reference's own (tests/test_gpu_radon_tiled.py).
__global__ void __launch_bounds__(256) ramp_exact_kernel(const float* __restrict__ x, float* __restrict__ out, int N) {
  DINVK_DYN_SMEM(double, sm);
  const int ne = (N + 1) >> 1, no = N >> 1;      // even-index / odd-index sample counts
  double* xe = sm;                                // x[2a]
  double* xo = sm + ne;                           // x[2a+1]
  double* w = xo + no;                            // w[c] = -2 / (pi (2c+1))^2, c < ne
  const long long row = blockIdx.x;
  const float* src = x + row * N;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double v = (double)__ldg(src + i);
    if (i & 1) xo[i >> 1] = v; else xe[i >> 1] = v;
  }
  for (int c = threadIdx.x; c < ne; c += blockDim.x) {
    const double d = 3.14159265358979323846264338327950288 * (double)(2 * c + 1);
    w[c] = -2.0 / (d * d);
  }
  __syncthreads();
  float* dst = out + row * N;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    // a CTA sweep covers 256 consecutive n: lanes alternate parity; the two parities read different arrays, each with unit stride
    const int a = n >> 1;
    double acc;
    if ((n & 1) == 0) {   // out[2a] = xe[a]/2 + sum_c w[c] (xo[a-c-1] + xo[a+c])
      acc = 0.5 * xe[a];
      const int cmax = max(a, no - a);            // c < a for the left arm, c < no - a for the right arm
      for (int c = 0; c < cmax; ++c) {
        const double l = (c < a) ? xo[a - c - 1] : 0.0, r = (a + c < no) ? xo[a + c] : 0.0;
        acc = fma(l + r, w[c], acc);
      }
    } else {              // out[2a+1] = xo[a]/2 + sum_c w[c] (xe[a-c] + xe[a+c+1])
      acc = 0.5 * xo[a];
      const int cmax = max(a + 1, ne - a - 1);
      for (int c = 0; c < cmax; ++c) {
        const double l = (c <= a) ? xe[a - c] : 0.0, r = (a + c + 1 < ne) ? xe[a + c + 1] : 0.0;
        acc = fma(l + r, w[c], acc);
      }
    }
    dst[n] = (float)acc;
  }
}
static std::map<std::vector<int>, float*> g_boxresp;
// B[n] = sum_{m < N} 2 f[(n - m) mod L], n < N: the response of the filter to the indicator of the valid samples (fp64)
static int get_box_response(int N, int L, float** out) {
  int dev = 0;
#ifndef DINVK_EMUL
  cudaGetDevice(&dev);
#endif
  std::lock_guard<std::mutex> lk(g_ramp_mu);
  std::vector<int> key = {dev, N, L};
  auto it = g_boxresp.find(key);
  if (it != g_boxresp.end()) { *out = it->second; return 0; }
  std::vector<double> f(L, 0.0);
  f[0] = 0.25;
  {
    std::vector<double> nn;
    for (int v = 1; v < L / 2 + 1; v += 2) nn.push_back(v);
    for (int v = L / 2 - 1; v > 0; v -= 2) nn.push_back(v);
    size_t q = 0;
    for (int k = 1; k < L; k += 2) { const double d = 3.14159265358979323846264338327950288 * nn[q++]; f[k] = -1.0 / (d * d); }
  }
  // prefix sums of f over the circular index make every B[n] an O(1) difference
  std::vector<double> pre(2 * L + 1, 0.0);
  for (int i = 0; i < 2 * L; ++i) pre[i + 1] = pre[i] + f[i % L];
  std::vector<float> B(N);
  for (int n = 0; n < N; ++n) {
    // indices (n - m) mod L for m = 0..N-1  ==  the circular range [n - N + 1, n]
    const int lo = n - N + 1 + L, hi = n + L;  // in [0, 2L)
    B[n] = (float)(2.0 * (pre[hi + 1] - pre[lo]));
  }
  float* d = nullptr;
  if (cudaMalloc((void**)&d, sizeof(float) * (size_t)N) != cudaSuccess) return set_error(DINVK_ECUDA, "cudaMalloc of the box-response table failed");
  cudaMemcpy(d, B.data(), sizeof(float) * (size_t)N, cudaMemcpyHostToDevice);
  g_boxresp[key] = d;
  *out = d;
  return 0;
}
}  // namespace dinvk

// workspace: the mean-free copy of the sinogram (rows * N floats) + one mean per row; without it (null / too small) the rows
// are filtered as they are
extern "C" size_t dinvk_ramp_filter_workspace_bytes(int rows, int N) {
  return (size_t)std::max(rows, 0) * (size_t)std::max(N, 0) * 4 + (size_t)std::max(rows, 0) * 4 + 256;
}

extern "C" int dinvk_ramp_filter(const float* sino, float* out, int rows, int N, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  DINVK_CHECK_ARG(sino && out && rows >= 0 && N >= 1, "dinvk_ramp_filter: bad arguments");
  if (rows == 0) return DINVK_OK;
  static const bool use_fft = getenv("DINVK_RAMP_FFT") != nullptr;
  if (!use_fft && N <= 8192) {  // exact spatial evaluation in fp64 (see ramp_exact_kernel); shared memory: (N + (N+1)/2) doubles
    const size_t smem = sizeof(double) * ((size_t)N + (size_t)((N + 1) / 2) + 2);
    int rc0;
    if ((rc0 = allow_smem(ramp_exact_kernel, smem))) return rc0;
    DINVK_LAUNCH(ramp_exact_kernel, dim3((unsigned)rows), dim3(256), smem, stream, sino, out, N);
    return DINVK_POST_LAUNCH();
  }
  DINVK_CHECK_ARG(rows >= 2, "dinvk_ramp_filter: needs at least 2 rows (rows are filtered in pairs)");
  const int L = ramp_padded_len(N);
  FftPlan pl;
  TileCfg cfg;
  if (!make_fft_plan(L, &pl) || !row_cfg(pl, L, &cfg)) return set_error(DINVK_EUNSUPPORTED, "dinvk_ramp_filter: padded length %d too large", L);
  Tables tb;
  int rc;
  if ((rc = get_tables(L, 0, &tb))) return rc;
  float* mult = nullptr;
  if ((rc = get_ramp_table(L, &mult))) return rc;
  auto run = [&](const float* src, float* dst, int npairs) -> int {
    PassParams P = PassParams();
    P.B = npairs; P.H = 1; P.W = L; P.wv = N;
    P.src_nc = 1; P.src_div = 1; P.dst_nc = 1; P.ncoil = 1;
    P.p0 = src; P.a0 = 1.f; P.out = dst; P.e0 = 1.f;
    P.dir1 = -1; P.dir2 = +1;
    P.gmode = DINVK_G_MASK; P.g = mult; P.gsb = 0; P.gsc = 0; P.gsh = 0; P.g_after = 1;
    P.tw = tb.tw; P.pre = tb.pre; P.post = tb.post; P.plan = pack_plan(pl);
    return launch_pass(false, P, cfg, stream);
  };
  const bool mean_free = workspace && workspace_bytes >= dinvk_ramp_filter_workspace_bytes(rows, N) && rows <= 2147483647;
  const float* src = sino;
  float* means = nullptr;
  float* boxresp = nullptr;
  if (mean_free) {
    if ((rc = get_box_response(N, L, &boxresp))) return rc;
    float* xc = reinterpret_cast<float*>(workspace);
    means = xc + (size_t)rows * N;
    DINVK_LAUNCH(ramp_mean_sub_kernel, dim3((unsigned)rows), dim3(256), 0, stream, sino, xc, means, N);
    if ((rc = DINVK_POST_LAUNCH())) return rc;
    src = xc;
  }
  const int npairs = rows / 2;
  if ((rc = run(src, out, npairs))) return rc;
  if (rows & 1) {
    // odd count: re-filter the last two rows as a pair (row rows-2 is recomputed identically)
    const long long off = (long long)(rows - 2) * N;
    if ((rc = run(src + off, out + off, 1))) return rc;
  }
  if (mean_free) {
    DINVK_LAUNCH(ramp_add_box_kernel, dim3((unsigned)rows), dim3(256), 0, stream, out, means, boxresp, N);
    if ((rc = DINVK_POST_LAUNCH())) return rc;
  }
  return DINVK_OK;
}
