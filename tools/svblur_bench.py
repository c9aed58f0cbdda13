"""Time the space-varying blur (libdinvk `dinvk_svblur_fwd` / `dinvk_svblur_adj`) on the GPU.

Workloads, synthetic seeded inputs:
  (a) (32, 1, 1024, 1024), K in {4, 10, 16}, one 31 x 31 filter set shared over the batch, circular and valid padding;
  (b) (64, 3, 256, 256), K = 8, per-sample 31 x 31 filters, circular padding.
For each: A, A_adjoint and one 50-iteration CG `prox_l2` through `SpaceVaryingBlur`, timed with CUDA events (median of
--reps after a warm-up), and the reference's loop restated in torch on the same GPU (per k: multiply, pad, grouped
F.conv2d, accumulate; the adjoint is the vjp of that restatement, i.e. its conv_transpose2d + padding fold), in strict fp32
(TF32 off), with the relative L2 distance between the two.  Reported beside the times: the algorithmic flops
(2 K h w per output pixel), the algorithmic bytes (x, y and the multiplier planes as stored), and the share of the fp32
FMA peak, the binding roofline here.  The card name and power limit are read in the same run.

    python tools/svblur_bench.py [--quick] [--reps N]

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

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
FP32_FLOPS = 67e12         # H100 SXM data sheet, non-tensor FP32


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


def timed(fn, reps: int) -> tuple[float, object]:
    out = fn()  # warm-up
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2], out


def torch_A(x, w, h, padding):
    """product_convolution2d restated: per k, w_k . x, the reference conv2d (flip, F.pad, grouped F.conv2d), accumulate"""
    B, C, H, W = x.shape
    fh, fw = h.shape[-2:]
    out = 0.0
    for k in range(w.size(2)):
        t = w[:, :, k] * x
        f = torch.flip(h[:, :, k], dims=(-2, -1)).expand(B, C, fh, fw).reshape(B * C, 1, fh, fw)
        if padding != "valid":
            t = F.pad(t, (fw // 2, fw - 1 - fw // 2, fh // 2, fh - 1 - fh // 2), mode=padding)
        Ho, Wo = t.shape[-2] - fh + 1, t.shape[-1] - fw + 1
        out = out + F.conv2d(t.reshape(1, B * C, *t.shape[-2:]), f, groups=B * C).reshape(B, C, Ho, Wo)
    return out


def run_case(shape, K, fsize, padding, per_sample, dev, reps, cg_iters=50):
    import deepinv_b200 as dinv

    B, C, H, W = shape
    g = torch.Generator(device=dev).manual_seed(K * 100 + fsize)
    x = torch.randn(*shape, device=dev, generator=g)
    w = torch.rand(1, 1, K, H, W, device=dev, generator=g)
    w = w / w.sum(2, keepdim=True)
    h = torch.rand(B if per_sample else 1, 1, K, fsize, fsize, device=dev, generator=g)
    h = h / h.sum((-2, -1), keepdim=True)
    phys = dinv.physics.SpaceVaryingBlur(filters=h, multipliers=w, padding=padding, device=dev)
    with torch.no_grad():
        t_a, y = timed(lambda: phys.A(x), reps)
        t_at, at = timed(lambda: phys.A_adjoint(y), reps)
        z = torch.zeros_like(x)
        t_cg, _ = timed(lambda: phys.prox_l2(z, y, 0.5, max_iter=cg_iters, tol=1e-12), 1)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            t_ta, yr = timed(lambda: torch_A(x, w, h, padding), reps)
        _, vjp = torch.func.vjp(lambda t: torch_A(t, w, h, padding), x)
        with torch.no_grad():
            t_tat, (atr,) = timed(lambda: vjp(y), reps)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    npx_out = y.numel()
    flops = 2 * K * fsize * fsize * npx_out
    byts = 4 * (x.numel() + y.numel() + w.numel())
    t_flop, t_hbm = flops / FP32_FLOPS * 1e3, byts / HBM_BYTES_PER_S * 1e3
    return {
        "shape": list(shape), "K": K, "filter": [fsize, fsize], "filters_per_sample": per_sample, "padding": padding,
        "A_ms": round(t_a, 3), "At_ms": round(t_at, 3), f"cg{cg_iters}_prox_ms": round(t_cg, 2),
        "torch_A_ms": round(t_ta, 3), "torch_At_ms": round(t_tat, 3),
        "speedup_A": round(t_ta / t_a, 2), "speedup_At": round(t_tat / t_at, 2),
        "rel_l2_A_vs_torch": rel(y, yr), "rel_l2_At_vs_torch": rel(at, atr),
        "gflop": round(flops / 1e9, 2), "mbytes": round(byts / 1e6, 1), "flop_per_byte": round(flops / byts, 1),
        "bound": "FP32" if t_flop >= t_hbm else "HBM", "bound_ms": round(max(t_flop, t_hbm), 3),
        "share_of_fp32_peak_A": round(t_flop / t_a, 3), "share_of_fp32_peak_At": round(t_flop / t_at, 3),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="one case of each workload")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("svblur_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card": card(), "cases": []}
    cases = [((32, 1, 1024, 1024), K, 31, pad, False) for K in ((10,) if a.quick else (4, 10, 16)) for pad in ("circular", "valid")]
    cases.append(((64, 3, 256, 256), 8, 31, "circular", True))
    for c in cases:
        res["cases"].append(run_case(*c, dev, a.reps))
        print(json.dumps(res["cases"][-1]), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
