// spectral_pipe.cuh — persistent, bulk-copy-pipelined spectral kernels for 256x256 images (included by spectral.cu).
//
// Same arithmetic as the tile passes in spectral.cu / spectral_fast.cuh (radix-16 Stockham stages, fp64-generated
// twiddles), restructured around what bounds the operator (DESIGN.md §4.1):
//
//   * HBM latency: the old passes kept < 40 KB per SM in flight (load -> barrier -> transform -> store inside each
//     CTA).  Here every kernel is persistent (2 CTAs per SM, static round-robin over tiles) and its tiles arrive by
//     `cp.async.bulk` (TMA 1-D bulk copies completing on an mbarrier) into a shared-memory ring filled one tile ahead,
//     so the loads of tile i+1 are in flight while tile i is transformed and stored.
//   * issue slots: a 256x256 fp32 FFT needs about as many issue cycles as HBM cycles.  Signs of the centred
//     transform, the orthonormal scale and the conjugations of the inverse are folded into per-thread constants or
//     the twiddle tables; all indexing is compile-time; the forward -> multiplier -> inverse row pass keeps the
//     spectrum in registers between the two transforms (the bins a thread owns after the last forward stage,
//     {j + 16 r}, are exactly the inputs of its first inverse butterfly).
//   * no narrow column strips: the H-direction transform is split 256 = 16 x 16.  Pass 1 owns the 16 rows
//     {b + 16 a} of an image (1 KB contiguous segments), transforms them along W, does the a-butterfly of the
//     H-transform per column in registers, and writes the intermediate as [k_lo][b][w]; pass 2 reads 16 contiguous
//     intermediate rows (one 32 KB bulk copy), does the b-butterfly per column and stores 16 output rows.
//     Every global access is a >= 1 KB contiguous segment.
//
// Kernels:  sp_row_fused   out = e0 * F_W^-1( g(mask[w]) * F_W(a0 p0 + a1 p1) ) + e1 q0 + e2 q1     (line masks)
//           sp_pass1       planar rows -> W transform -> H stage 1 (+ twiddle) -> interleaved workspace
//           sp_pass2       workspace -> H stage 2 -> multiplier / epilogue -> planar rows
// Restricted to H = W = 256, single-coil planar (B,2,H,W) tensors; everything else takes the tile passes.
#pragma once
#include "fft_core.cuh"

namespace dinvk {
namespace sp {

constexpr int N = 256;
constexpr int NT = 256;                 // threads per CTA (row kernels): thread = (line, j), a warp owns two lines
constexpr int IMO = 272;                // offset of the imaginary row inside a staged line, floats
constexpr int LSTR = 560;               // staged line stride, floats: [re 256 | pad 16 | im 256 | pad 32]; 560 % 32 == 16, so
                                        // the two lines of a warp hit disjoint banks; reused as 280 float2 for the transpose
constexpr int STAGE_F = 16 * LSTR;      // floats per staged tile
constexpr int RLS = 273;                // work-buffer line stride, float2 (pad16 layout)
constexpr size_t ROW_SMEM = (size_t)2 * STAGE_F * 4 + 256 * 8 + 64;  // two staged tiles (lines double as work rows) + twiddles + barriers
constexpr int P2_NT = 256;
constexpr int P2_STAGES = 3;
constexpr int P2_TILE_F = 16 * 256 * 2;  // floats per workspace tile (16 rows of 256 interleaved complex)
constexpr size_t P2_SMEM = (size_t)P2_STAGES * P2_TILE_F * 4 + 128;

struct PipeParams {
  int B;
  const float* p0; const float* p1; float a0, a1;
  int gmode; const float* g; long long gsb, gsc, gsh; float gc; const float* gcb;
  const float* q0; const float* q1; float e0, e1, e2;
  float* out;
  float2* ws;
  const float2* tw;   // exp(-2 pi i k / 256), k = 0..255
  int inverse;        // pass1 / pass2: 0 forward, 1 inverse (by conjugation)
  int centered;
  int g_at_load;      // pass1 applies the multiplier to the source (A^T); pass2 applies it to the result (A)
};

#ifdef DINVK_EMUL
// TEST-ONLY host model of the mbarrier / bulk-copy primitives (tests/emul): one 64-bit word per barrier holding
// [phase:1 | init:15 | pending:16 | tx bytes:32]; a phase completes when every expected arrival has happened AND the expected
// bytes have landed, exactly like the hardware object; the bulk copy is a synchronous memcpy followed by complete_tx.
#define DINVK_SP_DYN_SMEM() unsigned char* sp_raw = reinterpret_cast<unsigned char*>(::emul::dyn_smem())
namespace mbemul {
inline uint64_t pack(uint64_t phase, uint64_t init, uint64_t pending, int32_t tx) {
  return (phase << 63) | (init << 48) | (pending << 32) | (uint64_t)(uint32_t)tx;
}
inline void update(uint64_t* bar, int darrive, int32_t dtx) {
  for (;;) {
    uint64_t o = __atomic_load_n(bar, __ATOMIC_SEQ_CST);
    uint64_t phase = o >> 63, init = (o >> 48) & 0x7fff, pending = (o >> 32) & 0xffff;
    int32_t tx = (int32_t)(uint32_t)o;
    pending -= (uint64_t)darrive;
    tx += dtx;
    if (pending == 0 && tx == 0) { phase ^= 1; pending = init; }
    const uint64_t n = pack(phase, init, pending, tx);
    if (__atomic_compare_exchange_n(bar, &o, n, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) return;
  }
}
}  // namespace mbemul
inline void mb_init(uint64_t* bar, uint32_t count) { __atomic_store_n(bar, mbemul::pack(0, count, count, 0), __ATOMIC_SEQ_CST); }
inline void mb_expect_tx(uint64_t* bar, uint32_t bytes) { mbemul::update(bar, 1, (int32_t)bytes); }
inline void mb_arrive(uint64_t* bar) { mbemul::update(bar, 1, 0); }
inline void mb_wait(uint64_t* bar, uint32_t parity) {
  while ((__atomic_load_n(bar, __ATOMIC_SEQ_CST) >> 63) == (uint64_t)(parity & 1)) std::this_thread::yield();
}
inline void griddep_wait() {}
inline void griddep_launch() {}
inline void fence_async_smem() {}
inline void fence_mbar_init() {}
inline void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  std::memcpy(dst, src, bytes);
  mbemul::update(bar, 0, -(int32_t)bytes);
}
#else
#define DINVK_SP_DYN_SMEM() extern __shared__ __align__(128) unsigned char sp_raw[]
__device__ __forceinline__ uint32_t s_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mb_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mb_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ void mb_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok) : "r"(s_u32(bar)), "r"(parity) : "memory");
  }
}
// programmatic dependent launch: the kernels are launched with programmatic stream serialization, so their prologue
// (barrier init, twiddle tables) overlaps the tail of the previous kernel; nothing that depends on earlier kernels is
// touched before griddep_wait() returns (= previous grids complete and visible)
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// 1-D bulk copy global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s_u32(dst)),
               "l"(src), "r"(bytes), "r"(s_u32(bar))
               : "memory");
}

#endif  // DINVK_EMUL

// multiplier transform applied to K raw mask values at once: the mode switch sits outside the element loop
template <int K>
__device__ __forceinline__ void gmap(int gmode, float (&m)[K], float c) {
  if (gmode == DINVK_G_SQ) {
#pragma unroll
    for (int i = 0; i < K; ++i) m[i] = m[i] * m[i];
  } else if (gmode == DINVK_G_INV_SQ_PLUS_C) {
#pragma unroll
    for (int i = 0; i < K; ++i) m[i] = 1.0f / (m[i] * m[i] + c);
  } else if (gmode == DINVK_G_PINV) {
#pragma unroll
    for (int i = 0; i < K; ++i) m[i] = m[i] > 1e-5f ? 1.0f / m[i] : 0.0f;
  }
}

// ---- W-direction transform of one line, thread = (line, j); the 16 threads of a line sit in one warp, so the exchange
// between the two radix-16 stages only needs __syncwarp -------------------------------------------------------------
// stage 1: butterfly of x[j + 16 r], autosort store wk[16 j + r] (pad16 -> 17 j + r)
__device__ __forceinline__ void w_stage1_store(float2 (&v)[16], float2* wk, int j) {
  Dft<16>::run(v);
  float2* w = wk + 17 * j;
#pragma unroll
  for (int r = 0; r < 16; ++r) w[r] = v[r];
}
// stage 2: inputs wk[j + 16 r] (pad16 -> j + 17 r) times tw[r], butterfly -> v[r] = X[j + 16 r]
template <class TW>
__device__ __forceinline__ void w_stage2(float2 (&v)[16], const float2* wk, int j, TW tw) {
  const float2* w = wk + j;
#pragma unroll
  for (int r = 0; r < 16; ++r) v[r] = w[17 * r];
#pragma unroll
  for (int r = 1; r < 16; ++r) v[r] = cmul(v[r], tw(r));
  Dft<16>::run(v);
}

// shared-memory carve-up of the row kernels.  A staged line (re | im planes of one row, LSTR floats) doubles as the line's
// work row of RLS float2: every lane of the owning warp reads its stage inputs before any lane stores (a __syncwarp apart).
struct RowSmem {
  float* in0;    // two staged tiles
  float2* tws;   // [r][j]: sign(r) * w256^(r j)   (sign = (-1)^r for centred transforms: the (-1)^n pre-phase)
  uint64_t* full;   // [2] bulk copies landed
  uint64_t* empty;  // [2] all 8 warps released the stage
};
__device__ __forceinline__ RowSmem carve_row(unsigned char* raw) {
  RowSmem s;
  s.in0 = reinterpret_cast<float*>(raw);
  s.tws = reinterpret_cast<float2*>(s.in0 + 2 * STAGE_F);
  s.full = reinterpret_cast<uint64_t*>(s.tws + 256);
  s.empty = s.full + 2;
  return s;
}
__device__ __forceinline__ void fill_tables(const RowSmem& s, const float2* __restrict__ tw, int centered, int tid) {
  const int r = tid >> 4, j = tid & 15;
  float2 t = __ldg(tw + ((r * j) & 255));
  if (centered && (r & 1)) { t.x = -t.x; t.y = -t.y; }
  s.tws[tid] = t;
}
__device__ __forceinline__ void init_row_barriers(const RowSmem& s) {
  mb_init(&s.full[0], 1); mb_init(&s.full[1], 1);
  mb_init(&s.empty[0], NT / 32); mb_init(&s.empty[1], NT / 32);
  fence_mbar_init();
}

// issue the 32 row copies (16 rows x 2 planes, 1 KB each) of one tile; called by warp 0 (all lanes)
__device__ __forceinline__ void issue_rows(float* dst, const float* src_img, long long plane_stride, int row0, int row_step,
                                           uint64_t* bar, int lane) {
  if (lane == 0) mb_expect_tx(bar, 32 * 1024);
  __syncwarp();
  const int plane = lane >> 4, row = lane & 15;
  bulk_g2s(dst + row * LSTR + plane * IMO, src_img + plane * plane_stride + (long long)(row0 + row * row_step) * N, 1024, bar);
}

// ---------------------------------------------------------------------------------------------------------------------
// fused row pass (line masks): one tile = 16 consecutive rows of one image.  No CTA-wide barrier in the tile loop: a warp
// carries its two lines through both transforms; stages are recycled through full / empty mbarriers.
// ---------------------------------------------------------------------------------------------------------------------
template <bool HAS_P1, int OCC>
__global__ void __launch_bounds__(NT, OCC) sp_row_fused(const PipeParams P) {
  DINVK_SP_DYN_SMEM();
  const RowSmem S = carve_row(sp_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int line = tid >> 4, j = tid & 15;
  const int ntiles = P.B * 16;
  constexpr long long HW = (long long)N * N;

  const int t0 = blockIdx.x;
  if (tid < 32) {  // first tile on its way before anything else
    if (tid == 0) init_row_barriers(S);
    griddep_wait();
    if (tid == 0) griddep_launch();
    __syncwarp();
    if (t0 < ntiles) issue_rows(S.in0, P.p0 + (long long)(t0 >> 4) * 2 * HW, HW, (t0 & 15) * 16, 1, &S.full[0], lane);
  }
  fill_tables(S, P.tw, P.centered, tid);
  __syncthreads();

  const float scale = 0.0625f;                                   // 1/sqrt(256)
  const float sj = (P.centered && (j & 1)) ? -1.0f : 1.0f;      // (-1)^k post-phase, k = j + 16 r
  const float fmid = sj * scale;                                 // after the forward transform
  // e1 * q0 with q0 the (unscaled) source itself: F^-1 (e0 g) F x + e1 x = F^-1 (e0 g + e1) F x — folded into the multiplier,
  // so the staged source is not needed after the first butterfly
  const bool fold = (P.q0 != nullptr) && (P.q0 == P.p0) && !HAS_P1 && P.a0 == 1.0f;
  const float g_scale = fold ? P.e0 : 1.0f, g_shift = fold ? P.e1 : 0.0f;
  const float fend = sj * scale * (fold ? 1.0f : P.e0);          // after the inverse transform (and the epilogue weight)
  const bool ldq0 = (P.q0 != nullptr) && !fold;  // rare: loaded inline in the final pass
  const bool ldq1 = P.q1 != nullptr;
  const float2* twj = S.tws + j;
  auto tw = [&](int r) { return twj[16 * r]; };

  int it = 0;
  for (int t = t0; t < ntiles; t += gridDim.x, ++it) {
    const int s = it & 1;
    const int img = t >> 4, h0 = (t & 15) * 16;
    const int tn = t + gridDim.x;
    if (tid < 32 && tn < ntiles) {  // refill the other stage once every warp has released it (its use in iteration it-1)
      if (it >= 1) mb_wait(&S.empty[s ^ 1], ((it - 1) >> 1) & 1);
      fence_async_smem();
      issue_rows(S.in0 + (s ^ 1) * STAGE_F, P.p0 + (long long)(tn >> 4) * 2 * HW, HW, (tn & 15) * 16, 1, &S.full[s ^ 1], lane);
    }
    mb_wait(&S.full[s], (it >> 1) & 1);
    float* sl = S.in0 + s * STAGE_F + line * LSTR;
    float2* wk = reinterpret_cast<float2*>(sl);

    float2 v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) v[r] = make_float2(sl[j + 16 * r], sl[IMO + j + 16 * r]);
    __syncwarp();  // the line has been read by all of its lanes: it is the work row from here on
    if (HAS_P1) {
      const float* g1 = P.p1 + (long long)img * 2 * HW + (long long)(h0 + line) * N + j;
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        v[r].x = P.a0 * v[r].x + P.a1 * __ldg(g1 + 16 * r);
        v[r].y = P.a0 * v[r].y + P.a1 * __ldg(g1 + HW + 16 * r);
      }
    } else if (P.a0 != 1.0f) {
#pragma unroll
      for (int r = 0; r < 16; ++r) { v[r].x *= P.a0; v[r].y *= P.a0; }
    }
    w_stage1_store(v, wk, j);
    __syncwarp();
    w_stage2(v, wk, j, tw);
    // multiplier g(mask[img, w = j + 16 r]), forward post-phase and scale, conjugation for the inverse-by-conjugation
    if (P.gmode != DINVK_G_NONE) {
      const float* gp = P.g + (long long)img * P.gsb + j;
      const float c = P.gcb ? __ldg(P.gcb + img) : P.gc;
      float m[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) m[r] = __ldg(gp + 16 * r);
      gmap<16>(P.gmode, m, c);
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        const float mf = (g_scale * m[r] + g_shift) * fmid;
        v[r].x *= mf; v[r].y *= -mf;
      }
    } else {
      const float mf = (g_scale + g_shift) * fmid;
#pragma unroll
      for (int r = 0; r < 16; ++r) { v[r].x *= mf; v[r].y *= -mf; }
    }
    __syncwarp();  // every lane has read its stage-2 inputs: the warp's work rows may be overwritten
    w_stage1_store(v, wk, j);
    __syncwarp();
    // the warp writes its own two lines: lane handles 8 x 128 bits, f = lane + 32 i -> (line of the pair, plane, column group)
    const long long gbase = (long long)img * 2 * HW + (long long)(h0 + 2 * warp) * N;
    float4 qb[OCC == 2 ? 8 : 1];
    if (OCC == 2 && ldq1) {  // register budget allows it: second epilogue operand issued before the last butterfly
#pragma unroll
      for (int i = 0; i < (OCC == 2 ? 8 : 1); ++i) {
        const int f = lane + 32 * i, lp = f >> 7, plane = (f >> 6) & 1, c4 = f & 63;
        qb[i] = __ldg(reinterpret_cast<const float4*>(P.q1 + gbase + plane * HW + lp * N + 4 * c4));
      }
    }
    w_stage2(v, wk, j, tw);
    __syncwarp();  // stage-2 inputs consumed: the work row becomes the planar output row
    // conj, post-phase, scale, e0 -> planar
#pragma unroll
    for (int r = 0; r < 16; ++r) { sl[j + 16 * r] = fend * v[r].x; sl[IMO + j + 16 * r] = -fend * v[r].y; }
    __syncwarp();
    {
      const float* sw2 = S.in0 + s * STAGE_F + (2 * warp) * LSTR;
      float* ob = P.out + gbase;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int f = lane + 32 * i, lp = f >> 7, plane = (f >> 6) & 1, c4 = f & 63;
        float4 o = *reinterpret_cast<const float4*>(sw2 + lp * LSTR + plane * IMO + 4 * c4);
        if (ldq0) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(P.q0 + gbase + plane * HW + lp * N + 4 * c4));
          o.x += P.e1 * a.x; o.y += P.e1 * a.y; o.z += P.e1 * a.z; o.w += P.e1 * a.w;
        }
        if (ldq1) {
          float4 b4;
          if (OCC == 2) b4 = qb[OCC == 2 ? i : 0];
          else b4 = __ldg(reinterpret_cast<const float4*>(P.q1 + gbase + plane * HW + lp * N + 4 * c4));
          o.x += P.e2 * b4.x; o.y += P.e2 * b4.y; o.z += P.e2 * b4.z; o.w += P.e2 * b4.w;
        }
        *reinterpret_cast<float4*>(ob + plane * HW + lp * N + 4 * c4) = o;
      }
    }
    __syncwarp();
    if (lane == 0) mb_arrive(&S.empty[s]);  // this warp is done with stage s
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 1: tile = rows {b + 16 a} of one image.  W transform (warp-local), transpose through the warp's own staged lines,
// one CTA barrier, then the a-butterfly of the H transform per column, twiddle w256^(b k_lo), store to
// ws[img][k_lo][b][w] (interleaved)
// ---------------------------------------------------------------------------------------------------------------------
template <bool HAS_P1, int OCC>
__global__ void __launch_bounds__(NT, OCC) sp_pass1(const PipeParams P) {
  DINVK_SP_DYN_SMEM();
  const RowSmem S = carve_row(sp_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int line = tid >> 4, j = tid & 15;
  const int ntiles = P.B * 16;
  constexpr long long HW = (long long)N * N;

  const int t0 = blockIdx.x;
  if (tid < 32) {
    if (tid == 0) init_row_barriers(S);
    griddep_wait();
    if (tid == 0) griddep_launch();
    __syncwarp();
    if (t0 < ntiles) issue_rows(S.in0, P.p0 + (long long)(t0 >> 4) * 2 * HW, HW, t0 & 15, 16, &S.full[0], lane);
  }
  fill_tables(S, P.tw, P.centered, tid);
  __syncthreads();

  const float sgn_im = P.inverse ? -1.0f : 1.0f;                  // conj of the source for the inverse-by-conjugation
  const float sw = (P.centered && (tid & 1)) ? -1.0f : 1.0f;      // (-1)^k_w post-phase of the W transform, column = tid
  float2 twr[OCC == 2 ? 16 : 1];  // OCC == 2: stage-2 twiddles of this thread kept in registers across tiles
  if (OCC == 2) {
#pragma unroll
    for (int r = 0; r < (OCC == 2 ? 16 : 1); ++r) twr[r] = S.tws[r * 16 + j];
  }
  const float2* twj = S.tws + j;
  auto tw = [&](int r) { return OCC == 2 ? twr[OCC == 2 ? r : 0] : twj[16 * r]; };

  int it = 0;
  for (int t = t0; t < ntiles; t += gridDim.x, ++it) {
    const int s = it & 1;
    const int img = t >> 4, b = t & 15;
    const int tn = t + gridDim.x;
    if (tid < 32 && tn < ntiles) {
      if (it >= 1) mb_wait(&S.empty[s ^ 1], ((it - 1) >> 1) & 1);
      fence_async_smem();
      issue_rows(S.in0 + (s ^ 1) * STAGE_F, P.p0 + (long long)(tn >> 4) * 2 * HW, HW, tn & 15, 16, &S.full[s ^ 1], lane);
    }
    mb_wait(&S.full[s], (it >> 1) & 1);
    float* stage = S.in0 + s * STAGE_F;
    float* sl = stage + line * LSTR;
    float2* wk = reinterpret_cast<float2*>(sl);
    const int h = b + 16 * line;

    float2 v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) v[r] = make_float2(sl[j + 16 * r], sl[IMO + j + 16 * r]);
    __syncwarp();  // the line has been read by all of its lanes: it is the work row from here on
    if (HAS_P1) {
      const float* g1 = P.p1 + (long long)img * 2 * HW + (long long)h * N + j;
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        v[r].x = P.a0 * v[r].x + P.a1 * __ldg(g1 + 16 * r);
        v[r].y = P.a0 * v[r].y + P.a1 * __ldg(g1 + HW + 16 * r);
      }
    } else if (P.a0 != 1.0f) {
#pragma unroll
      for (int r = 0; r < 16; ++r) { v[r].x *= P.a0; v[r].y *= P.a0; }
    }
    if (P.g_at_load && P.gmode != DINVK_G_NONE) {
      const float* gp = P.g + (long long)img * P.gsb + (long long)h * P.gsh + j;
      const float c = P.gcb ? __ldg(P.gcb + img) : P.gc;
      float m0[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) m0[r] = __ldg(gp + 16 * r);
      gmap<16>(P.gmode, m0, c);
      if (P.gsc == 0) {  // same multiplier on both planes (line masks)
#pragma unroll
        for (int r = 0; r < 16; ++r) { v[r].x *= m0[r]; v[r].y *= sgn_im * m0[r]; }
      } else {
        float m1[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) m1[r] = __ldg(gp + P.gsc + 16 * r);
        gmap<16>(P.gmode, m1, c);
#pragma unroll
        for (int r = 0; r < 16; ++r) { v[r].x *= m0[r]; v[r].y *= sgn_im * m1[r]; }
      }
    } else if (P.inverse) {
#pragma unroll
      for (int r = 0; r < 16; ++r) v[r].y = -v[r].y;
    }
    w_stage1_store(v, wk, j);
    __syncwarp();
    w_stage2(v, wk, j, tw);
    __syncwarp();  // stage-2 inputs consumed
    {
      float2* tl = wk + j;  // transpose through the line's work row
#pragma unroll
      for (int r = 0; r < 16; ++r) tl[17 * r] = v[r];  // bin j + 16 r -> pad16 index j + 17 r
    }
    __syncthreads();
    // column stage: thread = column w = tid, butterfly over a (the tile's lines)
    {
      const float2* cl = reinterpret_cast<const float2*>(stage) + tid + (tid >> 4);
#pragma unroll
      for (int a = 0; a < 16; ++a) v[a] = cl[a * (LSTR / 2)];
    }
    __syncwarp();
    if (lane == 0) mb_arrive(&S.empty[s]);  // stage s consumed by this warp
    Dft<16>::run(v);
    {
      // twiddle w256^(b k_lo), H pre-phase (-1)^h = (-1)^b and W post-phase (-1)^w folded into one complex factor
      const float sb = ((P.centered && (b & 1)) ? -1.0f : 1.0f) * sw;
      float2* o = P.ws + ((long long)img * 256 + b) * N + tid;
      o[0] = make_float2(sb * v[0].x, sb * v[0].y);
#pragma unroll
      for (int k = 1; k < 16; ++k) {
        float2 tk = __ldg(P.tw + ((b * k) & 255));  // uniform across the CTA
        tk.x *= sb; tk.y *= sb;
        o[(long long)k * 16 * N] = cmul(v[k], tk);
      }
    }
  }
}

// pass-2 work of one column: b-butterfly of the 16 intermediate rows held in u -> rows h = k_lo + 16 k of column `tid`,
// multiplier (A), scale, conjugation (inverse), epilogue, planar stores
__device__ __forceinline__ void p2_finish(const PipeParams& P, float2 (&u)[16], int img, int klo, int tid) {
  constexpr long long HW = (long long)N * N;
  const float s2 = 1.0f / 256.0f;
  const float sgn_im = P.inverse ? -1.0f : 1.0f;
  const bool mult = (P.gmode != DINVK_G_NONE) && !P.g_at_load;
  Dft<16>::run(u);
  // (-1)^h post-phase = (-1)^k_lo; scale 1/256; e0
  const float f = ((P.centered && (klo & 1)) ? -1.0f : 1.0f) * s2 * P.e0;
  const float fi = sgn_im * f;
  const long long obase = (long long)img * 2 * HW + (long long)klo * N + tid;
  if (mult) {  // A: multiplier on the k-space result, rows h = k_lo + 16 k
    const float c = P.gcb ? __ldg(P.gcb + img) : P.gc;
    const float* gp = P.g + (long long)img * P.gsb + (long long)klo * P.gsh + tid;
    if (P.gsh == 0) {  // multiplier independent of the row (line masks): one value per column
      float m[2] = {__ldg(gp), __ldg(gp + P.gsc)};
      gmap<2>(P.gmode, m, c);
#pragma unroll
      for (int k = 0; k < 16; ++k) { u[k].x *= m[0]; u[k].y *= m[1]; }
    } else {
      float m0[16], m1[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float* gk = gp + (long long)(16 * k) * P.gsh;
        m0[k] = __ldg(gk);
        m1[k] = __ldg(gk + P.gsc);
      }
      gmap<16>(P.gmode, m0, c);
      gmap<16>(P.gmode, m1, c);
#pragma unroll
      for (int k = 0; k < 16; ++k) { u[k].x *= m0[k]; u[k].y *= m1[k]; }
    }
  }
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const long long o = obase + (long long)k * 16 * N;
    float re = f * u[k].x, im = fi * u[k].y;
    if (P.q0) { re += P.e1 * __ldg(P.q0 + o); im += P.e1 * __ldg(P.q0 + o + HW); }
    if (P.q1) { re += P.e2 * __ldg(P.q1 + o); im += P.e2 * __ldg(P.q1 + o + HW); }
    P.out[o] = re;
    P.out[o + HW] = im;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 2: tile = ws[img][k_lo][0..15][*] (32 KB contiguous, one bulk copy).  b-butterfly per column -> rows
// h = k_lo + 16 k_hi, multiplier (A), scale, conjugation (inverse), epilogue, planar store.  256 threads, thread = column;
// 3-stage ring recycled through full / empty mbarriers (no CTA barrier in the loop).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(P2_NT, 2) sp_pass2(const PipeParams P) {
  DINVK_SP_DYN_SMEM();
  float* ring = reinterpret_cast<float*>(sp_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + P2_STAGES * P2_TILE_F);
  uint64_t* empty = full + P2_STAGES;
  const int tid = threadIdx.x, lane = tid & 31;
  const int ntiles = P.B * 16;
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < P2_STAGES; ++i) { mb_init(&full[i], 1); mb_init(&empty[i], P2_NT / 32); }
    fence_mbar_init();
    griddep_wait();
    griddep_launch();
#pragma unroll
    for (int i = 0; i < P2_STAGES - 1; ++i) {
      const int t = blockIdx.x + i * gridDim.x;
      if (t < ntiles) {
        mb_expect_tx(&full[i], P2_TILE_F * 4);
        bulk_g2s(ring + i * P2_TILE_F, P.ws + (long long)t * 16 * N, P2_TILE_F * 4, &full[i]);
      }
    }
  }
  __syncthreads();
  int it = 0;
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    const int s = it % P2_STAGES;
    const int img = t >> 4, klo = t & 15;
    {
      const int ahead = it + P2_STAGES - 1;
      const int tn = blockIdx.x + ahead * gridDim.x;
      if (tid < 32 && tn < ntiles) {
        const int sn = ahead % P2_STAGES;  // == (it - 1) % STAGES: last used in iteration it-1
        if (it >= 1) mb_wait(&empty[sn], ((it - 1) / P2_STAGES) & 1);
        if (lane == 0) {
          fence_async_smem();
          mb_expect_tx(&full[sn], P2_TILE_F * 4);
          bulk_g2s(ring + sn * P2_TILE_F, P.ws + (long long)tn * 16 * N, P2_TILE_F * 4, &full[sn]);
        }
        __syncwarp();
      }
    }
    mb_wait(&full[s], (it / P2_STAGES) & 1);
    float2 u[16];
    {
      const float2* src = reinterpret_cast<const float2*>(ring + s * P2_TILE_F) + tid;
#pragma unroll
      for (int b = 0; b < 16; ++b) u[b] = src[b * N];
    }
    __syncwarp();
    if (lane == 0) mb_arrive(&empty[s]);
    p2_finish(P, u, img, klo, tid);
  }
}

}  // namespace sp
}  // namespace dinvk
