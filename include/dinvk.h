/*
 * dinvk.h — C ABI of libdinvk.so, the sm_90a kernel library behind the
 * deepinv_b200 drop-in physics operators / optim steps / denoisers.
 *
 * The reference (deepinv v0.4.1) is pure Python over ATen: it has no FFI of its
 * own.  Each entry point below therefore names the reference *function* whose
 * body it replaces (file:line relative to the reference tree) — that is the
 * binding a maintainer would swap (see INTEGRATION.md for the ctypes stubs).
 *
 * Conventions
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer unless the
 *     name ends in _host.  The caller (PyTorch) owns every buffer including the
 *     workspace; the library allocates nothing per call.  The only allocations it
 *     ever makes are immutable per-size twiddle/phase tables, cached per device
 *     behind a mutex on first use (dinvk_fft_prepare() forces this ahead of a
 *     CUDA-graph capture).
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no call
 *     synchronises the device; all calls are graph-capturable after warm-up.
 *   - return value: 0 on success, a DINVK_E* code otherwise; the message is
 *     available from dinvk_last_error() (thread-local).  No C++ exception ever
 *     crosses this boundary.
 *   - images are fp32, batch-major.  "planar complex" means the reference's
 *     (B,2,H,W) layout: plane 0 real, plane 1 imaginary (deepinv/utils/mixins.py:148-156).
 */
#ifndef DINVK_H
#define DINVK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DINVK_VERSION 100

enum {
  DINVK_OK = 0,
  DINVK_EINVAL = 1,     /* bad argument (shape, null pointer, unsupported mode) */
  DINVK_EWORKSPACE = 2, /* workspace too small */
  DINVK_ECUDA = 3,      /* CUDA runtime / launch error */
  DINVK_EUNSUPPORTED = 4
};

int dinvk_version(void);
const char* dinvk_last_error(void);
/* number of kernel launches issued by this library since load (bench.py "gpu_launches") */
uint64_t dinvk_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Spectral ("decomposable") operators: MRI and BlurFFT
 * ------------------------------------------------------------------------------------------
 * One generic fused primitive covers every DecomposablePhysics method of the reference
 * (deepinv/physics/forward.py:1080-1252) for V = centred/plain orthonormal 2-D DFT:
 *
 *   u   = a0*p0 + a1*p1                           (prologue, planar complex, p1 optional)
 *   U   = F(u)            if fwd                  (2-D DFT, norm="ortho", centred like
 *                                                  deepinv/utils/mixins.py:158-180 when centered=1)
 *   U  <- g(mask) (.) U                           (pointwise multiplier, see DINVK_G_*)
 *   v   = F^-1(U)         if inv
 *   out = e0*v + e1*q0 + e2*q1                    (epilogue, q0/q1 optional)
 *
 * fwd=1,inv=0  : A          = mask (.) F x                    MRI.A        forward.py:1080-1095 + mri.py:100-101
 * fwd=0,inv=1  : A_adjoint  = F^-1 (mask (.) y)               MRI.A_adjoint forward.py:1097-1116; g=PINV gives A_dagger :1236-1252
 * fwd=1,inv=1  : A_adjoint_A (g=SQ), prox_l2 (g=INV_SQ_PLUS_C, forward.py:1212-1234), and the fused
 *                PGD data step z = x - gamma*(A^T A x - A^T y)  (optim_iterators/pgd.py:137-139 + data_fidelity.py:335-336)
 * fwd=0,inv=0  : plain elementwise (used for U/U_adjoint = identity paths)
 *
 * The mask is addressed as mask[b*mask_sb + ch*mask_sc + h*mask_sh + w] (element strides):
 *   (B,2,H,W) full mask: sb=2HW sc=HW sh=W;  batch-1 mask: sb=0;  column ("Cartesian line")
 *   mask stored as (B,1,1,W): sh=0, sc=0 — when the multiplier does not depend on h and is the same
 *   on both planes (a complex scalar per column) and fwd=inv=1, the H-direction transforms cancel
 *   and the library runs 1-D row transforms only (one pass over HBM).
 * For complex multipliers (BlurFFT, blur.py:639-692) `mask` points at interleaved (re,im) pairs
 * addressed as ((float2*)mask)[b*mask_sb + h*mask_sh + w] and mask_sc is ignored.
 */
enum {
  DINVK_G_NONE = 0,          /* U unchanged                                  */
  DINVK_G_MASK = 1,          /* U_ch *= m_ch                                 */
  DINVK_G_SQ = 2,            /* U_ch *= m_ch^2               (A^T A)         */
  DINVK_G_INV_SQ_PLUS_C = 3, /* U_ch /= (m_ch^2 + c)         (prox_l2)       */
  DINVK_G_PINV = 4,          /* U_ch *= (m_ch > 1e-5 ? 1/m_ch : 0) (A_dagger) */
  DINVK_G_CMUL = 5,          /* U *= h      (complex multiplier)             */
  DINVK_G_CMUL_CONJ = 6      /* U *= conj(h)                                 */
};

typedef struct dinvk_spectral_args {
  int32_t B, H, W;     /* number of complex images, height, width                         */
  int32_t fwd, inv;    /* which transforms run (see above)                                 */
  int32_t centered;    /* 1: fftshift(fft(ifftshift(.))) (MRI); 0: plain fft (BlurFFT)     */
  int32_t gmode;       /* DINVK_G_*                                                        */
  const float* p0;     /* planar (B,2,H,W)                                                 */
  const float* p1;     /* planar or NULL                                                   */
  float a0, a1;
  const float* mask;   /* multiplier or NULL when gmode==NONE                              */
  int64_t mask_sb, mask_sc, mask_sh;
  float c;             /* constant for INV_SQ_PLUS_C (=1/gamma)                            */
  const float* c_batch;/* optional per-image constants (B floats); overrides c             */
  const float* q0;     /* planar or NULL                                                   */
  const float* q1;     /* planar or NULL                                                   */
  float e0, e1, e2;
  float* out;          /* planar (B,2,H,W)                                                 */
  /* multi-coil extension (deepinv/physics/mri.py:254-324); ncoil<=1 disables it.
   * B counts coil images (= batch*ncoil).  With ncoil>1:
   *   coil_mode 1 (A):         u[b,n] = S[b,n] * x[b]; p0 is (batch,2,H,W); out is (batch,2,ncoil,H,W)
   *   coil_mode 2 (A_adjoint): p0 is (batch,2,ncoil,H,W); out[b] = sum_n conj(S[b,n]) * v[b,n] (batch,2,H,W)
   *   coil_mode 3 (rss):       out[b] = sqrt(sum_n |v[b,n]|^2) as (batch,1,H,W)
   * coil maps are interleaved complex64 (batch|1, ncoil, H, W); coil_sb = batch stride in complex elements (0 if shared) */
  int32_t ncoil, coil_mode;
  const float* coil_maps;
  int64_t coil_sb;
} dinvk_spectral_args;

size_t dinvk_spectral_workspace_bytes(int B, int H, int W);
int dinvk_spectral(const dinvk_spectral_args* args, void* workspace, size_t workspace_bytes, void* stream);
/* build + cache the per-size tables now (call once before graph capture) */
int dinvk_fft_prepare(int n, int centered);

/* 3-D: the same operator with F the centred (or plain) orthonormal 3-D DFT of contiguous (D,H,W) volumes
 * (deepinv/physics/mri.py:11-163 with three_d=True, MultiCoilMRI.A / A_adjoint on (B,2,N,D,H,W), mri.py:254-324).
 * `args` means what it means for dinvk_spectral, with every "H,W" read as "D,H,W": B counts complex volumes, p0 / p1 / q0 /
 * q1 / out are planar (B,2,D,H,W), and the mask is addressed as mask[b*mask_sb + ch*mask_sc + (d*H + h)*mask_sh + w]
 * ((B,2,D,H,W) full mask: sb=2DHW sc=DHW sh=W).  Coils: coil_mode 0 uses no maps (see below); coil_mode 1..3 has the
 * meaning above for any ncoil >= 1 (a single coil included), with x / out (batch,2,D,H,W), y (batch,2,ncoil,D,H,W), the
 * rss volume (batch,1,D,H,W) and interleaved complex64 maps (batch|1, ncoil, D, H, W), coil_sb in complex elements.
 * coil_mode 0 with ncoil = N > 1 transforms a plain stack of N volumes per sample: p0 / p1 / q0 / q1 / out are all
 * (batch,2,N,D,H,W), no maps, and the mask is the sample's (b = volume / N), shared by its N volumes.
 * Sizes as dinvk_spectral: each axis is a power-of-two or mixed radix 2/3/4/5/8/16 tile pass; an axis with another prime
 * factor (or past the tile budget) takes an O(N^2) DFT, and the call then runs unfused (elementwise prologue / epilogue
 * around the three axis transforms); D*H*W < 2^31.
 * No launch for B == 0. */
size_t dinvk_spectral3d_workspace_bytes(int B, int D, int H, int W);
int dinvk_spectral3d(const dinvk_spectral_args* args, int D, void* workspace, size_t workspace_bytes, void* stream);

/* Ramp filter of filtered back-projection (deepinv/physics/functional/radon.py:79-162): `rows` (>= 2)
 * signals of length N (contiguous, one per row — the angle-major sinogram memory (B*C*A, P)), each
 * zero-padded to L = max(64, 2^ceil(log2(2N))), multiplied by 2*rfft(f) with f the reference's spatial ramp
 * kernel (built by the library in double from the closed form, :151-162), inverse-transformed, cropped to N.
 * Default (N <= 8192): the SAME linear filter evaluated exactly in the spatial domain with fp64 accumulation (the padded
 * circular convolution is a linear one on the N valid samples and the kernel has a closed form) — the result is the filter to
 * fp32 rounding, where an fp32 FFT leaves ~4e-6 (a sinogram row is ~100x larger than its filtered version).  DINVK_RAMP_FFT=1
 * selects the FFT form; there, with a workspace of dinvk_ramp_filter_workspace_bytes(rows, N) the row means are removed before the fp32 transform and their
 * exact response (mean x filter(box), built in double) is added back: the result is the same linear filter, an order of
 * magnitude closer to its exact value (the transform's rounding noise scales with the norm of what it is given). */
size_t dinvk_ramp_filter_workspace_bytes(int rows, int N);
int dinvk_ramp_filter(const float* sino, float* out, int rows, int N,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Elementwise / reduction helpers used by the optim steps and CG
 * (deepinv/optim/optim_iterators/*.py axpy algebra, optim/linear/conjugate_gradient.py:47-66,
 *  optim/linear/utils.py:6-26 batched dot)
 * ------------------------------------------------------------------------------------------ */
/* out = a*x + b*y + c*z   (y, z optional: pass NULL) ; n elements */
int dinvk_axpbypcz(float* out, const float* x, float a, const float* y, float b,
                   const float* z, float c, int64_t n, void* stream);
/* per-sample scaled update: out[b,i] = x[b,i] + sa * s[b] * y[b,i]   (CG x/r/p updates; s on device) */
int dinvk_batched_axpy(float* out, const float* x, const float* y, const float* s, float sa,
                       int B, int64_t n_per, void* stream);
/* per-sample real dot products: out[b] = sum_i x[b,i]*y[b,i]  (fp32 in, fp32 accumulate per
 * thread, fp64 across the block; deterministic: no atomics) */
int dinvk_batched_dot(float* out, const float* x, const float* y, int B, int64_t n_per,
                      void* workspace, size_t workspace_bytes, void* stream);
size_t dinvk_batched_dot_workspace_bytes(int B, int64_t n_per);
/* CG scalar update on device, one thread per sample (conjugate_gradient.py:55-66).  `done_flag` is a
 * sticky int32 the caller zeroes once per solve:
 *   mode 0: alpha = rsold / (pAp + eps) -> out0, forced to 0 once done_flag is set (iterations issued
 *           after convergence leave x and r untouched, so the host may poll the flag lazily)
 *   mode 1: beta  = rsnew / (rsold + eps) -> out0, and done_flag <- 1 when all(rsnew < tol2*bnorm2)
 *           (bnorm2 entries <= 0 are replaced by 1, conjugate_gradient.py:51) */
int dinvk_cg_scalars(int mode, float* out0, const float* num, const float* den, float eps,
                     const float* bnorm2, float tol2, int32_t* all_done_flag, int B, void* stream);

/* DDRM spectral-domain update (deepinv/sampling/diffusion.py:163-222), n real elements; the mask is
 * broadcast over the batch (index i % mask_n, the reference requires a batch-1 mask, :173).
 *   init=1 : first draw (:175-190): y_bar is normalised in place by (|mask|+eps) where |mask|>sigma_noise,
 *            x_bar_out = mean + std * noise / sqrt(2) with sigma_t = sigmas[0]
 *   init=0 : step t (:196-220) with c_sig = sqrt(1-eta^2) * sigmas[t], sigma_prev = sigmas[t-1] */
int dinvk_ddrm_update(float* x_bar_out, const float* x_bar, const float* x_bar_prev, float* y_bar,
                      const float* mask, const float* noise, int64_t n, int64_t mask_n, float sigma_t,
                      float sigma_prev, float sigma_noise, float eta, float etab, float c_sig, float eps,
                      int init, void* stream);

/* interleaved complex (B, n_per) [re, im, ...] -> planar (B, 2, n_per): raw k-space as stored in MRI files -> the operators'
 * planar layout (deepinv/utils/mixins.py:148-156 from_torch_complex, as used by datasets/fastmri.py:475-478) */
int dinvk_interleaved_to_planar(const float* in, float* out, int B, int64_t n_per, void* stream);

/* ------------------------------------------------------------------------------------------
 * Radon (deepinv/physics/functional/radon.py:252-342 forward, autograd transpose of it
 * = tomography.py:322-342, IRadon back-projection radon.py:396-450)
 * ------------------------------------------------------------------------------------------
 * x    : (BC, W, W) fp32 contiguous (square images)
 * sino : (BC, A, P) fp32, ANGLE-major — the reference returns exactly this memory as the
 *        non-contiguous view (B,C,P,A) (radon.py:291-293); the host wrapper re-views it.
 * P = ceil(sqrt(2)*W) (circle=0) or W (circle=1); scale multiplies the result (1/operator_norm).
 * cos_t / sin_t: 2*A floats each — the A fp32 values cos(theta_t), followed by their A low-order parts
 *        (cos = hi + lo, evaluated in fp64 on the host from the fp32 angles; pass zeros for plain fp32 tables).
 *        dinvk_radon_fwd / dinvk_radon_adj evaluate the sample coordinates in fp64 from hi + lo (closer to the exact
 *        operator than the reference's fp32 affine_grid); dinvk_iradon_bp / dinvk_fanbeam read the first A values only.
 */
int dinvk_radon_fwd(const float* x, float* sino, int BC, int W, int P, int A, int circle,
                    const float* cos_t, const float* sin_t, float scale, void* stream);
/* exact transpose of dinvk_radon_fwd (same weights; tiled path: per-tile 32-bit fixed-point accumulation, csrc/radon.cu) */
int dinvk_radon_adj(const float* sino, float* x, int BC, int W, int P, int A, int circle,
                    const float* cos_t, const float* sin_t, float scale, void* stream);
/* IRadon back-projection (adjoint_via_backprop=False / FBP geometry), sinogram sampled bilinearly
 * in (angle, detector) exactly as grid_sample(align_corners=True) does; output (BC,W,W) */
int dinvk_iradon_bp(const float* sino, float* x, int BC, int W, int P, int A, int circle,
                    const float* cos_t, const float* sin_t, float scale, void* stream);

/* fan-beam projector (adjoint = 0: image (BC,W,W) -> sinogram (BC,A,D)) and its exact transpose (adjoint = 1), replacing
 * grid_sample over fan_beam_grid + sum (deepinv/physics/functional/radon.py:16-52, 252-309 with fan_beam=True) and its
 * autograd transpose (tomography.py:322-342).  G = grid size (W if circle else ceil(sqrt(2) W)), D = detector pixels;
 * the sample of ray j at step i is R_t(x_i, y_j * ((half_len * (x_i + src)) / den)) with x = linspace(-1,1,G),
 * y = linspace(-1,1,D); half_len, src, den are the reference's scaled fp32 constants (0.5 * detector_length,
 * source_radius, source_radius + detector_radius).  The transpose accumulates with fp32 atomics. */
int dinvk_fanbeam(const float* in, float* out, int BC, int W, int G, int D, int A, int circle,
                  const float* cos_t, const float* sin_t, float half_len, float src, float den, float scale,
                  int adjoint, void* stream);

/* ------------------------------------------------------------------------------------------
 * Blur (deepinv/physics/functional/convolution.py:42-164 conv2d / conv_transpose2d)
 * ------------------------------------------------------------------------------------------
 * x (B,C,H,W), filter (FB,FC,h,w) with FB in {1,B}, FC in {1,C}; padding: 0 valid, 1 circular,
 * 2 replicate, 3 reflect, 4 constant(zero).  fwd output is (B,C,H-h+1,W-w+1) for valid else (B,C,H,W).
 * adj input is that shape, output (B,C,H,W).
 */
enum { DINVK_PAD_VALID = 0, DINVK_PAD_CIRCULAR = 1, DINVK_PAD_REPLICATE = 2, DINVK_PAD_REFLECT = 3, DINVK_PAD_CONSTANT = 4 };
int dinvk_blur_fwd(const float* x, const float* filt, float* y, int B, int C, int H, int W,
                   int FB, int FC, int h, int w, int padding, void* stream);
/* transpose; replicate/reflect need a workspace for the zero-extended (H+h-1, W+w-1) image that is folded back */
size_t dinvk_blur_adj_workspace_bytes(int B, int C, int H, int W, int h, int w, int padding);
int dinvk_blur_adj(const float* y, const float* filt, float* x, int B, int C, int H, int W,
                   int FB, int FC, int h, int w, int padding,
                   void* workspace, size_t workspace_bytes, void* stream);

/* 3-D blur (deepinv/physics/functional/convolution.py:333-438 conv3d / conv_transpose3d with _apply_transpose_padding
 * :689-758; deepinv/physics/blur.py:496-561, Blur.A / A_adjoint on 5-D tensors).
 * x (B,C,D,H,W), filter (FB,FC,d,h,w) with FB in {1,B}, FC in {1,C}; paddings as dinvk_blur_fwd, applied per axis with the same
 * origin (d/2, h/2, w/2).  fwd output is (B,C,D-d+1,H-h+1,W-w+1) for valid else (B,C,D,H,W); adj input is that shape, output
 * (B,C,D,H,W).  h and w are limited as in dinvk_blur_fwd (DINVK_EUNSUPPORTED past it), d is not.  One launch (two for the
 * replicate / reflect adjoint), no atomics. */
int dinvk_blur3d_fwd(const float* x, const float* filt, float* y, int B, int C, int D, int H, int W,
                     int FB, int FC, int d, int h, int w, int padding, void* stream);
/* transpose; replicate/reflect need a workspace for the zero-extended (D+d-1, H+h-1, W+w-1) volume that is folded back */
size_t dinvk_blur3d_adj_workspace_bytes(int B, int C, int D, int H, int W, int d, int h, int w, int padding);
int dinvk_blur3d_adj(const float* y, const float* filt, float* x, int B, int C, int D, int H, int W,
                     int FB, int FC, int d, int h, int w, int padding,
                     void* workspace, size_t workspace_bytes, void* stream);

/* Space-varying blur, the product convolution y = sum_{k<K} h_k * (w_k . x) and its adjoint
 * x = sum_k w_k . (h_k^T * y) (deepinv/physics/functional/product_convolution.py:10-68).
 * x (B,C,H,W), multipliers (MB,MC,K,H,W), filters (FB,FC,K,h,w); MB, FB in {1,B} and MC, FC in {1,C}
 * independently.  Shapes and paddings otherwise as dinvk_blur_fwd / dinvk_blur_adj; the adjoint needs
 * the same workspace as dinvk_blur_adj.  One launch (two for the replicate / reflect adjoint), no atomics. */
int dinvk_svblur_fwd(const float* x, const float* mult, const float* filt, float* y, int B, int C, int H, int W,
                     int MB, int MC, int FB, int FC, int K, int h, int w, int padding, void* stream);
size_t dinvk_svblur_adj_workspace_bytes(int B, int C, int H, int W, int h, int w, int padding);
int dinvk_svblur_adj(const float* y, const float* mult, const float* filt, float* x, int B, int C, int H, int W,
                     int MB, int MC, int FB, int FC, int K, int h, int w, int padding,
                     void* workspace, size_t workspace_bytes, void* stream);

/* Tiled space-varying blur (deepinv/physics/blur.py:871-1192, TiledSpaceVaryingBlur.A / A_adjoint; multipliers from
 * deepinv/physics/functional/tiled_product_convolution.py:105-143), valid padding:
 *   y = sum_k Wt_k . (h_k * x),  x = sum_k h_k^T * (Wt_k . y).
 * x (B,C,H,W) in both directions, y (B,C,H-h+1,W-w+1), filters (FB,FC,K,h,w) with FB in {1,B}, FC in {1,C}, multipliers
 * (K,P1,P2) shared over B and C.  The image is padded at the bottom / right to the compatible size of patch (P1,P2) and
 * stride (s1,s2) (deepinv/utils/_tiling.py:27-46), which holds nr x nc patches; patch k = r*nc + c covers rows
 * [r*s1, r*s1+P1) and columns [c*s2, c*s2+P2), and Wt_k is its multiplier placed there and cropped to y, which starts at
 * (h/2, w/2).  DINVK_EINVAL unless nr*nc == K and 1 <= s <= P.  One launch, no workspace, no atomics. */
int dinvk_tiled_svblur_fwd(const float* x, const float* mult, const float* filt, float* y, int B, int C, int H, int W,
                           int FB, int FC, int K, int h, int w, int P1, int P2, int s1, int s2, void* stream);
int dinvk_tiled_svblur_adj(const float* y, const float* mult, const float* filt, float* x, int B, int C, int H, int W,
                           int FB, int FC, int K, int h, int w, int P1, int P2, int s1, int s2, void* stream);

/* MATLAB-bicubic resize (deepinv/physics/functional/imresize.py:222-372, imresize_matlab with kernel 'cubic' and reflect
 * padding; DownsamplingMatlab.A, deepinv/physics/blur.py:1195-1261) and its exact transpose (DownsamplingMatlab.A_adjoint).
 * Per plane y = M_H x M_W^T: x (BC,H,W) -> y (BC,Ho,Wo).  Each axis is a banded matrix given by tables the caller builds:
 *   forward  : base (n_out) int32, the first (unreflected) tap of each output, and weights (n_out, k) fp32; output o reads
 *              input base[o] + t for t < k, reflected as j < 0 -> -1 - j, j >= n -> 2n - 1 - j (the caller guarantees that
 *              the band reaches at most n samples past either edge);
 *   transpose: the same matrix transposed, CSR by input index: ptr (n_in + 1), and per entry the output index (int32, sorted
 *              ascending within a row) and weight (fp32).  Taps that reflection folds onto one input stay separate entries.
 * kw and scale_w (Wo / W as the resize defines it, > 0) size the shared-memory band of a tile.  Each output sums its taps in
 * table order with every product and sum rounded separately: one launch, no workspace, no atomics, bitwise reproducible.
 * BC == 0 launches nothing. */
int dinvk_resize_fwd(const float* x, float* y, int BC, int H, int W, int Ho, int Wo, const int* base_h, const float* wt_h,
                     int kh, const int* base_w, const float* wt_w, int kw, double scale_w, void* stream);
int dinvk_resize_adj(const float* y, float* x, int BC, int H, int W, int Ho, int Wo, const int* ptr_h, const int* out_h,
                     const float* wt_h, const int* ptr_w, const int* out_w, const float* wt_w, int kw, double scale_w,
                     void* stream);

/* ------------------------------------------------------------------------------------------
 * Denoiser convolutions (deepinv/models/drunet.py:200-210,323-433; dncnn.py:116-131)
 * ------------------------------------------------------------------------------------------
 * fp32 reference-precision path (CUDA cores), NCHW:
 *   kind 0: 3x3 stride 1 zero-pad 1;  kind 1: 2x2 stride 2 (downsample_strideconv);
 *   kind 2: transposed 2x2 stride 2 (upsample_convtranspose, weight (Cin,Cout,2,2))
 *   out = act( conv(x [+ xadd]) + bias ) + res ; act: 0 none, 1 ReLU (applied before the residual)
 */
int dinvk_conv_f32(const float* x, const float* xadd, const float* weight, const float* bias,
                   const float* res, float* out, int B, int Cin, int Cout, int H, int W,
                   int kind, int act, void* stream);

/* backward of dinvk_conv_f32 (training through the denoiser inside unfolded / deep-equilibrium models,
 * deepinv/unfolded/unfolded.py:9-120, deep_equilibrium.py:70-139; replaces ATen's convolution_backward):
 *   data gradient: the forward entry itself — kind 0 with the transposed + flipped filter, kind 1 <-> kind 2;
 *   weight (+ bias) gradient: dweight has the forward weight's layout, dbias (Cout) optional; both are zeroed
 *   here and accumulated with fp32 atomics (summation order is not deterministic);
 *   x [+ xadd] is the forward input, gout the gradient w.r.t. the pre-residual output (after dinvk_relu_bwd
 *   when the forward had act = 1).  B, Cin, Cout, H, W are the FORWARD call's arguments. */
int dinvk_conv_f32_wgrad(const float* x, const float* xadd, const float* gout, float* dweight, float* dbias,
                         int B, int Cin, int Cout, int H, int W, int kind, void* stream);
/* gin = gout * [out > 0] : backward of the fused ReLU, `out` being the forward output */
int dinvk_relu_bwd(const float* gout, const float* out, float* gin, long long n, void* stream);

/* bf16 tensor-core path (wgmma implicit GEMM, TMA-fed), NHWC bf16 activations:
 *   x (B,H,W,Cin) bf16, weight (Cout, 9*Cin) bf16 K-major with k = (ky*3+kx)*Cin + c,
 *   out (B,H,W,Cout) bf16;  out = act(conv3x3(x) + bias) + res + res2   (bias fp32 (Cout) optional;
 *   res/res2 optional, bf16 NHWC; res2 carries the U-Net skip that the reference adds before the next
 *   stage, drunet.py:206-209).  Cin, Cout multiples of 64 (the host pads the head layer's input channels). */
int dinvk_conv3x3_bf16(const void* x, const void* weight, const float* bias, const void* res, const void* res2,
                       void* out, int B, int H, int W, int Cin, int Cout, int act, void* stream);
/* network tail: Cout <= 16 real output channels (weight padded to 16 rows), result written as fp32 NCHW
 *   out_nchw = conv3x3(x) + bias + add_nchw   (add_nchw optional: DnCNN's "+ x", dncnn.py:138) */
int dinvk_conv3x3_bf16_tail(const void* x, const void* weight16, const float* bias, const float* add_nchw,
                            float* out_nchw, int B, int H, int W, int Cin, int Cout, void* stream);
/* network head: 3x3 convolution straight from the reference's NCHW fp32 image to 64 NHWC bf16 channels
 *   x_nchw (B,C,H,W) fp32; has_fill appends one constant channel (DRUNet's noise-level map, drunet.py:190-200:
 *   fill_batch[b] if non-null else fill_scalar); CT = C + has_fill in 1..4;
 *   weight64 (64, 64) bf16 with k = (ky*3+kx)*CT + c, zero padded to 64;  out = act(conv3x3(x) + bias)  */
int dinvk_conv3x3_head_bf16(const float* x_nchw, const void* weight64, const float* bias, void* out_nhwc, int B,
                            int C, int H, int W, float fill_scalar, const float* fill_batch, int has_fill,
                            int act, void* stream);
/* layout converters between the reference's NCHW fp32 and the tensor-core NHWC bf16 layout
 *   nchw_to_nhwc: out[b,h,w,c] = c < C ? in[b,c,h,w] : (c == C ? fill[b] or fill_scalar : 0), c < Cpad
 *   nhwc_to_nchw: out[b,c,h,w] = in[b,h,w,c] (+ add[b,c,h,w] if add), c < C */
int dinvk_nchw_f32_to_nhwc_bf16(const float* in, void* out, int B, int C, int H, int W, int Cpad,
                                float fill_scalar, const float* fill_batch, int has_fill, void* stream);
int dinvk_nhwc_bf16_to_nchw_f32(const void* in, const float* add, float* out, int B, int C, int H, int W,
                                int Cpad, void* stream);
/* 2x2 stride-2 down / transposed-up as GEMMs on the same layout:
 *   down: x (B,H,W,Cin) -> out (B,H/2,W/2,Cout), weight (Cout, 4*Cin) k=(dy*2+dx)*Cin+c
 *   up  : x (B,H,W,Cin) (+xadd) -> out (B,2H,2W,Cout), weight (4*Cout, Cin) row=(dy*2+dx)*Cout+co */
int dinvk_conv2x2_down_bf16(const void* x, const void* xadd, const void* weight, void* out,
                            int B, int H, int W, int Cin, int Cout, void* stream);
int dinvk_conv2x2_up_bf16(const void* x, const void* xadd, const void* weight, void* out,
                          int B, int H, int W, int Cin, int Cout, void* stream);


/* fp32-grade tensor-core path (split-operand wgmma implicit GEMM, TMA-fed; replaces the same ATen / cuDNN calls as
 * dinvk_conv_f32: deepinv/models/drunet.py:200-263,323-433, dncnn.py:116-140) — every fp32 value v travels as a pair
 * (hi, lo) of narrow values, products hi*hi + hi*lo + lo*hi are accumulated in fp32 and drained to registers every `window`
 * pipeline steps (0 = library default).  Two formats (`fmt`):
 *   fmt 0 "split16"  (fp32 words):  hi = tf32(v), lo = v - hi;               kind::tf32;  any fp32 range
 *   fmt 1 "split32h" (fp16 words):  hi = fp16(v), lo = fp16((v - hi) 2^11);  kind::f16 (twice the channels per MMA, half the
 *         bytes);  |v| < 65504 — an activation beyond it sets *overflow_flag (sticky, may be null) and the tail kernel of a
 *         network whose flag is set writes NaN: loud, never silent
 * Activation layout: (B,H,W,C/CH,2,CH) words, CH = 16 (fmt 0) / 32 (fmt 1), [..,0,:] = hi, [..,1,:] = lo.
 * Weights: per 64 output channels 128 K-major rows [W_hi (64); W_lo (64)] in the same word type (fmt 1: W_lo scaled 2^11):
 *   kind 0 (3x3, pad 1): (2*Cout, 9*Cin), k = (ky*3+kx)*Cin + c
 *   kind 1 (2x2 stride 2): (2*Cout, 4*Cin), k = (dy*2+dx)*Cin + c;  out (B,H/2,W/2,Cout)
 *   kind 2 (transposed 2x2 stride 2): (8*Cout, Cin), GEMM column = (dy*2+dx)*Cout + co;  out (B,2H,2W,Cout)
 *   out = act(conv(x) + bias) + res + res2 (res/res2: same layout, kind 0 only).  Cin % (2 CH) == 0, Cout % 64 == 0. */
int dinvk_conv_tc32(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                    int B, int H, int W, int Cin, int Cout, int kind, int act, int window, int fmt, int* overflow_flag,
                    void* stream);
/* kind 0 with halo reuse (the body layers): one (16+8) x (16+2)-position activation slab per CH-channel block serves all
 * nine taps.  weight: "slab pack" (2*Cout, 10*Cin), column ((c/CH * 5 + tap/2) * 2 + tap%2) * CH + c%CH (tap 9 = zeros);
 * `window` counted in channel blocks of 9 taps (0 = default: one block = 18 full-scale MMA accumulations per window).  Cin % CH == 0, Cout % 64 == 0. */
int dinvk_conv_tc32_slab(const void* x, const void* weight, const float* bias, const void* res, const void* res2,
                         void* out, int B, int H, int W, int Cin, int Cout, int act, int window, int fmt,
                         int* overflow_flag, void* stream);
/* head: NCHW fp32 image (+ optional constant noise-level channel) -> split layout; weight (Cout, C + has_fill, 3, 3) fp32 */
int dinvk_conv_tc32_head(const float* x_nchw, const float* weight, const float* bias, void* out, int B, int C, int H,
                         int W, int Cout, float fill_scalar, const float* fill_batch, int has_fill, int act, int fmt,
                         int* overflow_flag, void* stream);
/* tail: split layout -> NCHW fp32, Cout <= 4;  out = conv3x3(x) + bias + add_nchw;  weight (Cout, Cin, 3, 3) fp32;
 * NaN everywhere if *overflow_flag is set */
int dinvk_conv_tc32_tail(const void* x, const float* weight, const float* bias, const float* add_nchw,
                         float* out_nchw, int B, int H, int W, int Cin, int Cout, int fmt, const int* overflow_flag,
                         void* stream);
/* layout converters split <-> NCHW fp32 (C % CH == 0); called with H' = D*H they convert NDHWC split volumes <-> NCDHW */
int dinvk_split16_to_nchw(const void* in, float* out, int B, int C, int H, int W, int fmt, void* stream);
int dinvk_nchw_to_split16(const float* in, void* out, int B, int C, int H, int W, int fmt, void* stream);

/* 3-D denoiser convolutions (DRUNet(dim=3): deepinv/models/drunet.py with Conv3d / ConvTranspose3d), forward only.
 * fp32 CUDA-core path, NCDHW:  kind 0: 3x3x3 stride 1 zero-pad 1, weight (Cout,Cin,3,3,3);  kind 1: 2x2x2 stride 2 (D, H, W
 *   even), weight (Cout,Cin,2,2,2);  kind 2: transposed 2x2x2 stride 2, weight (Cin,Cout,2,2,2);
 *   out = act(conv(x [+ xadd]) + bias) + res, as dinvk_conv_f32. */
int dinvk_conv3d_f32(const float* x, const float* xadd, const float* weight, const float* bias, const float* res,
                     float* out, int B, int Cin, int Cout, int D, int H, int W, int kind, int act, void* stream);
/* split-operand wgmma path on NDHWC split volumes (B,D,H,W,C/CH,2,CH), formats and weight rows as dinvk_conv_tc32:
 *   kind 0 (3x3x3, pad 1): (2*Cout, 27*Cin), k = ((kz*3+ky)*3+kx)*Cin + c
 *   kind 1 (2x2x2 stride 2): (2*Cout, 8*Cin), k = (dz*4+dy*2+dx)*Cin + c;  out (B,D/2,H/2,W/2,Cout)
 *   kind 2 (transposed 2x2x2 stride 2): (16*Cout, Cin), GEMM column = (dz*4+dy*2+dx)*Cout + co;  out (B,2D,2H,2W,Cout)
 *   out = act(conv(x) + bias) + res + res2 (kind 0 only).  Cin % (2 CH) == 0, Cout % 64 == 0. */
int dinvk_conv3d_tc32(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                      int B, int D, int H, int W, int Cin, int Cout, int kind, int act, int window, int fmt,
                      int* overflow_flag, void* stream);
/* 3-D head: NCDHW fp32 volume (+ optional constant noise-level channel) -> split NDHWC; weight (Cout, C + has_fill, 3,3,3) */
int dinvk_conv3d_tc32_head(const float* x_ncdhw, const float* weight, const float* bias, void* out, int B, int C, int D,
                           int H, int W, int Cout, float fill_scalar, const float* fill_batch, int has_fill, int act,
                           int fmt, int* overflow_flag, void* stream);
/* 3-D tail: split NDHWC -> NCDHW fp32, Cout <= 4;  out = conv3x3x3(x) + bias + add_ncdhw;  NaN if *overflow_flag is set */
int dinvk_conv3d_tc32_tail(const void* x, const float* weight, const float* bias, const float* add_ncdhw,
                           float* out_ncdhw, int B, int D, int H, int W, int Cin, int Cout, int fmt,
                           const int* overflow_flag, void* stream);

/* ------------------------------------------------------------------------------------------
 * Total variation (2-D, images (B,C,H,W) fp32; gradient fields (B,C,H,W,2), component 0 vertical)
 * ------------------------------------------------------------------------------------------
 * TV prox by over-relaxed Chambolle-Pock, TVDenoiser.forward / TVL1Denoiser (deepinv/models/tv.py:86-151, 238-239).
 * Each launch runs up to `dinvk_tv_block` iterations of tv.py:131-137 on two ping-pong state buffers
 * (x2_a, u2_a) / (x2_b, u2_b), reads the per-sample lambd (B,) from device memory and applies the reference's break
 * test (it > 1 and ||x_prev - x2|| / ||x2 + 1e-12|| < crit over the whole tensor, tv.py:139-145) for every iteration
 * without a host synchronisation.  The state of the solve lives in a 64-byte control block at the head of the workspace,
 * int32 [ticket, it_done, cur, status, replay_n, conv_j1, -, -]:
 *   it_done  iterations whose result is in buffer `cur` (0: a, 1: b);  status 0 running, 1 finished, 2 replay pending;
 *   conv_j1  1 + the sub-iteration of the converging launch at which the test passed (0: it never passed).
 * If the test passes before the last iteration of a launch, the next launch recomputes the iterations up to the break
 * from that launch's input into its output (status 2), so the result is bitwise the state after the reference's break
 * iteration.  Launches issued after the solve finished return at entry.  first != 0 zeroes the control block (call it
 * that way once per prox, with (x2_a, u2_a) holding the start state); each call enqueues n_launch launches.
 * mode 0: isotropic dual projection u / max(|u| / lambd, 1) (TV), 1: per-component clamp to [-lambd, lambd] (TV-L1).
 * tau, rho: the reference's python floats; sigma = 1 / tau / 8 and 1 + tau are formed in double and rounded once. */
int dinvk_tv_prox(const float* y, float* x2_a, float* u2_a, float* x2_b, float* u2_b, const float* lambd, int B, int C,
                  int H, int W, int n_it_max, float crit, double tau, double rho, int mode, int first, int n_launch,
                  void* workspace, size_t workspace_bytes, void* stream);
size_t dinvk_tv_prox_workspace_bytes(int B, int C, int H, int W);
/* the library's compile-time tile edge T and iterations per launch K of dinvk_tv_prox (host pointers) */
int dinvk_tv_block(int* tile_host, int* iters_host);
/* one-launch stencils: op 0 nabla (tv.py:153-181) in (B,C,H,W) -> out (B,C,H,W,2); op 1 nabla_adjoint (tv.py:183-218)
 * (B,C,H,W,2) -> (B,C,H,W); op 2 the TV subgradient nabla_adjoint(Dx / |Dx|), 0 where |Dx| = 0 (TVPrior.grad,
 * deepinv/optim/prior.py:544-572); op 3 TGV's epsilon (deepinv/models/tgv.py:229-270) (B,C,H,W,2) -> (B,C,H,W,4),
 * backward differences with component 2i + j = d(field i)/d(axis j), zero first row / column; op 4 its adjoint
 * epsilon_adjoint (tgv.py:272-312) (B,C,H,W,4) -> (B,C,H,W,2).  Ops 3 and 4 need the (…,4) field 16-byte aligned
 * and the (…,2) field 8-byte aligned. */
int dinvk_tv_stencil(int op, const float* in, float* out, int B, int C, int H, int W, void* stream);

/* TGV prox by over-relaxed Chambolle-Pock, TGVDenoiser.forward (deepinv/models/tgv.py:93-213, 2-D).  Each launch runs
 * up to `dinvk_tgv_block` iterations of tgv.py:149-160 on two ping-pong state buffers (x2_a, r2_a, u2_a) /
 * (x2_b, r2_b, u2_b): x2 (B,C,H,W), r2 (B,C,H,W,2) 8-byte aligned, u2 (B,C,H,W,4) 16-byte aligned.  tl1 = tau * lambda1
 * and l2 = lambda2 are (B,) fp32 on the device, formed by the caller as the reference forms them (tgv.py:124-143, 77).
 * The break test is the reference's, it > 1 and ||x_prev - x2|| / (||x2|| + 1e-12) < crit over the whole tensor
 * (tgv.py:162-170), evaluated on the device with the control block, replay and `first` / n_launch protocol of
 * dinvk_tv_prox.  tau, rho: the reference's attributes (0.01, 1.99); sigma = 1 / tau / 72 and 1 + tau are formed in
 * double and rounded once.  The workspace (8-byte aligned) holds the control block and the per-CTA sums. */
int dinvk_tgv_prox(const float* y, float* x2_a, float* r2_a, float* u2_a, float* x2_b, float* r2_b, float* u2_b,
                   const float* tl1, const float* l2, int B, int C, int H, int W, int n_it_max, float crit, double tau,
                   double rho, int first, int n_launch, void* workspace, size_t workspace_bytes, void* stream);
size_t dinvk_tgv_prox_workspace_bytes(int B, int C, int H, int W);
/* the library's compile-time tile edge T and iterations per launch K of dinvk_tgv_prox (host pointers) */
int dinvk_tgv_block(int* tile_host, int* iters_host);
/* per-sample TV value (TVPrior.fn / TVL1Prior.fn, prior.py:507-522, 595-611): out[b] = sum |Dx| with the 2-norm over
 * the two differences (mode 0) or the 1-norm (mode 1); fp64 across the block and the chunks, deterministic */
int dinvk_tv_fn(float* out, const float* x, int mode, int B, int C, int H, int W, void* workspace,
                size_t workspace_bytes, void* stream);
size_t dinvk_tv_fn_workspace_bytes(int B, int C, int H, int W);

#ifdef __cplusplus
}
#endif
#endif /* DINVK_H */
