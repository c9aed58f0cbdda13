"""Time the tiled space-varying blur (libdinvk `dinvk_tiled_svblur_fwd` / `dinvk_tiled_svblur_adj`) on the GPU.

Workloads, synthetic seeded inputs:
  (a) (32, 1, 1024, 1024), patch 128, stride 64 (K = 225), per-sample 31 x 31 motion-blur PSFs (`TiledBlurGenerator`);
  (b) (64, 3, 256, 256), patch 64, stride 32 (K = 49), one 15 x 15 PSF set shared over the batch.
For each: A, A_adjoint and one 50-iteration CG `prox_l2` through `TiledSpaceVaryingBlur`, timed with CUDA events (median and
range of --reps after a warm-up), and the reference's per-patch algorithm restated in torch on the same GPU (unfold into halo'd
patches, grouped F.conv2d or 2-D FFT products, multiply, fold; the adjoint is the vjp of the direct restatement), in strict
fp32 (TF32 off), with the relative L2 distance between the two.  Work: the algorithmic FMAs (per output pixel, the patches
covering it times h w), the FMAs the kernels execute (per warp of 8 x 64 output pixels, the terms whose rows it meets times
the tile's terms along columns, times 512 h w), and the share of the fp32 FMA peak.  Card name and power limit are read in the
same run.

    python tools/tiledsv_bench.py [--reps N]

Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import torch  # noqa: E402

import tiledsv_oracle as O  # noqa: E402

FP32_FLOPS = 67e12  # H100 SXM data sheet, non-tensor FP32
HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit": "not read"}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            name, pl, clk = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
            info.update(name=name, power_limit=pl, max_sm_clock=clk)
    except (OSError, subprocess.SubprocessError):
        pass
    return info


def timed(fn, reps: int):
    out = fn()  # warm-up
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    times.sort()
    return {"median": round(times[len(times) // 2], 3), "min": round(times[0], 3), "max": round(times[-1], 3)}, out


def _range(lo, hi, p, s, n):
    """(first, count) of the patches along one dimension whose span [k s, k s + p) meets [lo, hi] (the kernels' term_range)"""
    a = 0 if lo - p + 1 <= 0 else (lo - p + 1 + s - 1) // s
    return a, (0 if lo > hi else max(0, min(n - 1, hi // s) - a + 1))


def _span(lo, hi, p, s, n):
    return _range(lo, hi, p, s, n)[1]


def work(H, W, fh, fw, patch, stride):
    """(algorithmic, executed forward, executed adjoint) FMAs per (b, c) plane, the kernels' tile and warp enumeration"""
    (P1, P2), (s1, s2) = patch, stride
    nr, nc = O.num_patches(H, W, patch, stride)
    ai, aj, Ho, Wo = fh // 2, fw // 2, H - fh + 1, W - fw + 1
    cov_r = [_span(i + ai, i + ai, P1, s1, nr) for i in range(Ho)]
    cov_c = [_span(j + aj, j + aj, P2, s2, nc) for j in range(Wo)]
    algo = sum(cov_r) * sum(cov_c) * fh * fw
    ex = []
    for fwd in (True, False):
        d_i, d_j = (ai, aj) if fwd else (32, 32)
        Hout, Wout = (Ho, Wo) if fwd else (H, W)
        tot = 0
        for tj in range((Wout + d_j + 63) // 64):
            oj = 64 * tj - d_j
            if fwd:
                cols = _span(max(oj, 0) + aj, min(oj + 64, Wout) - 1 + aj, P2, s2, nc)
            else:  # output columns [lo, hi] read y columns [lo - (w - 1), hi]
                cols = _span(max(max(oj, 0) - (fw - 1), 0) + aj, min(min(oj + 64, Wout) - 1, Wo - 1) + aj, P2, s2, nc)
            for ti in range((Hout + d_i + 63) // 64):
                oi = 64 * ti - d_i
                if fwd:
                    r0, rows = _range(max(oi, 0) + ai, min(oi + 64, Hout) - 1 + ai, P1, s1, nr)
                else:
                    r0, rows = _range(max(max(oi, 0) - (fh - 1), 0) + ai, min(min(oi + 64, Hout) - 1, Ho - 1) + ai, P1, s1, nr)
                if rows == 0 or cols == 0:
                    continue
                for wgrp in range(8):  # a warp: 8 output rows
                    wr = oi + 8 * wgrp
                    for r in range(r0, r0 + rows):
                        lo, hi = (r * s1 - ai, r * s1 - ai + P1) if fwd else (r * s1 - ai, r * s1 - ai + P1 + fh - 1)
                        if not (wr + 8 <= lo or wr >= hi):
                            tot += cols * 512 * fh * fw
        ex.append(tot)
    return algo, ex[0], ex[1]


def run_case(shape, patch, stride, fsize, per_sample, dev, reps, cg_iters=50):
    import deepinv_b200 as dinv
    from deepinv_b200.physics.generator import MotionBlurGenerator, TiledBlurGenerator

    B, C, H, W = shape
    g = torch.Generator(device=dev).manual_seed(H + fsize)
    x = torch.rand(*shape, device=dev, generator=g)
    gen = TiledBlurGenerator(MotionBlurGenerator((fsize, fsize), device=dev), patch_size=patch, stride=stride, device=dev)
    h = gen.step(batch_size=B if per_sample else 1, img_size=(H, W), seed=1)["filters"]
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=h, patch_size=patch, stride=stride, device=dev)
    with torch.no_grad():
        t_a, y = timed(lambda: phys.A(x), reps)
        t_at, at = timed(lambda: phys.A_adjoint(y), reps)
        t_cg, _ = timed(lambda: phys.prox_l2(torch.zeros_like(x), y, 0.5, max_iter=cg_iters, tol=1e-12), 2)
    w = phys.multipliers
    pp, ss = (patch, patch), (stride, stride)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            t_ta, yr = timed(lambda: O.tiledsv_A_patches(x, w, h, pp, ss), reps)
            t_tf, yf = timed(lambda: O.tiledsv_A_patches(x, w, h, pp, ss, fft=True), reps)
        _, vjp = torch.func.vjp(lambda t: O.tiledsv_A_patches(t, w, h, pp, ss), x)
        with torch.no_grad():
            t_tat, (atr,) = timed(lambda: vjp(y), reps)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    algo, ex_f, ex_a = (B * C * n for n in work(H, W, fsize, fsize, pp, ss))
    byts = 4 * (x.numel() + y.numel() + h.numel())
    t_flop, t_hbm = 2 * algo / FP32_FLOPS * 1e3, byts / HBM_BYTES_PER_S * 1e3
    return {
        "shape": list(shape), "patch": patch, "stride": stride, "K": h.shape[2], "filter": [fsize, fsize],
        "filters_per_sample": per_sample, "A_ms": t_a, "At_ms": t_at, f"cg{cg_iters}_prox_ms": t_cg,
        "torch_A_conv_ms": t_ta, "torch_A_fft_ms": t_tf, "torch_At_conv_ms": t_tat,
        "speedup_A_vs_conv": round(t_ta["median"] / t_a["median"], 2), "speedup_A_vs_fft": round(t_tf["median"] / t_a["median"], 2),
        "speedup_At_vs_conv": round(t_tat["median"] / t_at["median"], 2),
        "rel_l2_A_vs_torch_conv": rel(y, yr), "rel_l2_A_vs_torch_fft": rel(y, yf), "rel_l2_At_vs_torch_conv": rel(at, atr),
        "algorithmic_gfma": round(algo / 1e9, 2), "executed_gfma_A": round(ex_f / 1e9, 2), "executed_gfma_At": round(ex_a / 1e9, 2),
        "executed_over_algorithmic_A": round(ex_f / algo, 3), "executed_over_algorithmic_At": round(ex_a / algo, 3),
        "mbytes": round(byts / 1e6, 1), "bound": "FP32" if t_flop >= t_hbm else "HBM", "bound_ms": round(max(t_flop, t_hbm), 3),
        "share_of_fp32_peak_A": round(t_flop / t_a["median"], 3), "share_of_fp32_peak_At": round(t_flop / t_at["median"], 3),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--work-only", action="store_true", help="print the FMA counts of the two workloads and exit (no GPU)")
    a = ap.parse_args()
    cases = [((32, 1, 1024, 1024), 128, 64, 31, True), ((64, 3, 256, 256), 64, 32, 15, False)]
    if a.work_only:
        for shape, p, s, f, _ in cases:
            algo, ef, ea = work(*shape[2:], f, f, (p, p), (s, s))
            print(json.dumps({"shape": shape, "patch": p, "stride": s, "filter": f, "fwd": round(ef / algo, 3), "adj": round(ea / algo, 3)}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("tiledsv_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card(), "cases": []}
    for c in cases:
        res["cases"].append(run_case(*c, dev, a.reps))
        print(json.dumps(res["cases"][-1]), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
