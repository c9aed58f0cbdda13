// conv_tc32_model.cu — TEST-ONLY.  The CUDA-core kernels of deepinv_b200/csrc/conv_tc32.cu (head, tail, layout converters: the same
// source, compiled for the host) plus a SCALAR MODEL of its tensor-core layers, so that the package's fp32-grade denoiser engines
// (deepinv_b200/models/tc_engine.py: packing orders, residual / skip wiring, overflow flag) can run end to end on the host emulation.
// The model implements the C-ABI contract of dinvk_conv_tc32 / dinvk_conv_tc32_slab — operands as (hi, lo) pairs, the three products
// hi*hi + hi*lo + lo*hi accumulated per output, bias / ReLU / residual epilogue through the product's own store_split / add_split —
// with plain loops; it shares NO code with the wgmma kernels and says nothing about them (those are tested on the H100,
// tests/test_gpu_tc32.py).  Never linked into libdinvk.so.
#include "../../deepinv_b200/csrc/conv_tc32.cu"

namespace {
using namespace dinvk::t32;

template <class F>
inline double elem_val(const typename F::elem* p, int part) {   // part 0: hi, 1: lo (weighted)
  return part == 0 ? (double)(float)p[0] : (double)(float)p[F::CH] * (double)F::CORR;
}
// (hi, lo) of channel c of a split-layout pixel (C channels)
template <class F>
inline void act_pair(const typename F::elem* pix, int c, double& hi, double& lo) {
  const typename F::elem* p = pix + (c / F::CH) * 2 * F::CH + (c % F::CH);
  hi = (double)(float)p[0];
  lo = (double)(float)p[F::CH] * (double)F::CORR;
}
// (hi, lo) of logical row n, column k of a packed weight matrix (per 64 rows [hi (64); lo (64)], K columns)
template <class F>
inline void w_pair(const typename F::elem* w, long long K, int n, long long k, double& hi, double& lo) {
  const long long r = (long long)(n / 64) * 128 + n % 64;
  hi = (double)(float)w[r * K + k];
  lo = (double)(float)w[(r + 64) * K + k] * (double)F::CORR;
}

// kind 0: 3x3 (slab_order: the halo kernel's K order), 1: 2x2 stride 2, 2: transposed 2x2 stride 2
template <class F>
int model_conv(const void* xv, const void* wv, const float* bias, const void* resv, const void* res2v, void* outv, int B, int H, int W,
               int Cin, int Cout, int kind, bool slab_order, int relu, int* flag) {
  using E = typename F::elem;
  const E* x = static_cast<const E*>(xv);
  const E* w = static_cast<const E*>(wv);
  const E* res = static_cast<const E*>(resv);
  const E* res2 = static_cast<const E*>(res2v);
  E* out = static_cast<E*>(outv);
  const int Ho = kind == 1 ? H / 2 : (kind == 2 ? 2 * H : H), Wo = kind == 1 ? W / 2 : (kind == 2 ? 2 * W : W);
  const long long K = kind == 0 ? (slab_order ? 10LL * Cin : 9LL * Cin) : (kind == 1 ? 4LL * Cin : (long long)Cin);
  bool bad = false;
  for (int b = 0; b < B; ++b)
    for (int yo = 0; yo < Ho; ++yo)
      for (int xo = 0; xo < Wo; ++xo) {
        E* opix = out + (((long long)b * Ho + yo) * Wo + xo) * Cout * 2;
        for (int c0 = 0; c0 < Cout; c0 += F::CH) {
          float v[F::CH];
          for (int i = 0; i < F::CH; ++i) {
            const int co = c0 + i;
            double main = 0.0, corr = 0.0;
            auto acc = [&](const E* ipix, int n, long long kbase, bool slab_cols, int tap) {
              for (int c = 0; c < Cin; ++c) {
                double ah, al, wh, wl;
                act_pair<F>(ipix, c, ah, al);
                const long long k = slab_cols ? ((long long)((c / F::CH) * 5 + tap / 2) * 2 + tap % 2) * F::CH + c % F::CH : kbase + c;
                w_pair<F>(w, K, n, k, wh, wl);
                main += ah * wh;
                corr += ah * wl + al * wh;
              }
            };
            if (kind == 0) {
              for (int tap = 0; tap < 9; ++tap) {
                const int yy = yo + tap / 3 - 1, xx = xo + tap % 3 - 1;
                if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
                acc(x + (((long long)b * H + yy) * W + xx) * Cin * 2, co, (long long)tap * Cin, slab_order, tap);
              }
            } else if (kind == 1) {
              for (int tap = 0; tap < 4; ++tap)
                acc(x + (((long long)b * H + 2 * yo + (tap >> 1)) * W + 2 * xo + (tap & 1)) * Cin * 2, co, (long long)tap * Cin, false, tap);
            } else {
              const int tap = (yo & 1) * 2 + (xo & 1);
              acc(x + (((long long)b * H + yo / 2) * W + xo / 2) * Cin * 2, tap * Cout + co, 0, false, 0);
            }
            float r = (float)(main + corr);
            if (bias) r += bias[co];
            if (relu) r = fmaxf(r, 0.f);
            v[i] = r;
          }
          const long long o = (((long long)b * Ho + yo) * Wo + xo) * Cout * 2 + (long long)(c0 / F::CH) * 2 * F::CH;
          if (res) add_split<F>(res + o, v);
          if (res2) add_split<F>(res2 + o, v);
          bad |= store_split<F>(opix + (c0 / F::CH) * 2 * F::CH, v);
        }
      }
  if (bad && flag) *flag |= 1;
  return DINVK_OK;
}
}  // namespace

extern "C" int dinvk_conv_tc32(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out, int B,
                               int H, int W, int Cin, int Cout, int kind, int act, int /*window*/, int fmt, int* overflow_flag, void* /*stream*/) {
  using namespace dinvk::t32;
  DINVK_CHECK_ARG(x && weight && out && kind >= 0 && kind <= 2, "conv_tc32 (model): bad arguments");
  DINVK_CHECK_ARG(Cout % 64 == 0 && Cout >= 64, "conv_tc32: Cout=%d must be a multiple of 64", Cout);
  DINVK_CHECK_ARG(kind == 0 || (!res && !res2), "conv_tc32: residual inputs are for kind 0 only");
  ::dinvk::count_launch();
  DINVK_FMT_DISPATCH(fmt, model_conv<FmtTF32>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, kind, false, act, overflow_flag),
                     model_conv<FmtF16>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, kind, false, act, overflow_flag));
}

extern "C" int dinvk_conv_tc32_slab(const void* x, const void* weight, const float* bias, const void* res, const void* res2, void* out,
                                    int B, int H, int W, int Cin, int Cout, int act, int /*window*/, int fmt, int* overflow_flag,
                                    void* /*stream*/) {
  using namespace dinvk::t32;
  DINVK_CHECK_ARG(x && weight && out, "conv_tc32_slab (model): null pointer");
  DINVK_CHECK_ARG(Cout % 64 == 0 && Cout >= 64, "conv_tc32_slab: Cout=%d must be a multiple of 64", Cout);
  ::dinvk::count_launch();
  DINVK_FMT_DISPATCH(fmt, model_conv<FmtTF32>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, 0, true, act, overflow_flag),
                     model_conv<FmtF16>(x, weight, bias, res, res2, out, B, H, W, Cin, Cout, 0, true, act, overflow_flag));
}
