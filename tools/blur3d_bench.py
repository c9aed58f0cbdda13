"""Time the 3-D blur (libdinvk `dinvk_blur3d_fwd` / `dinvk_blur3d_adj`, `Blur` on (B, C, D, H, W) volumes) on the GPU.

Workloads, synthetic seeded inputs at sizes a microscopy user runs:
  (a) (4, 1, 64, 256, 256) with a 15 x 15 x 15 and a 21 x 31 x 31 PSF, circular and valid padding;
  (b) (1, 3, 32, 256, 256) with per-channel 11 x 21 x 21 PSFs, circular;
  (c) a 50-iteration CG `prox_l2` on (a)'s 15^3 circular blur.
For A and A^T: ms per call (CUDA events, median and range of --reps after a warm-up), the share of the fp32 FMA data-sheet peak
counted on algorithmic FMAs (d h w per output voxel), and the torch restatement of the reference's conv3d on the same GPU in
strict fp32 (TF32 off: flip, F.pad, grouped F.conv3d; the transpose is the vjp of that restatement, i.e. conv_transpose3d plus
the padding's fold), with the relative L2 distance between the two.  Card name and power limit are read in the same run.

    python tools/blur3d_bench.py [--reps N] [--out FILE]

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

FP32_FMA_PER_S = 67e12 / 2  # H100 SXM data sheet, non-tensor FP32 (FLOP/s; one FMA = 2 FLOP)


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


def torch_conv3d(x, k, pad):
    """the reference's conv3d (deepinv/physics/functional/convolution.py:333-392) in torch: flip, pad, grouped conv3d"""
    B, C = x.shape[:2]
    d, h, w = k.shape[-3:]
    kk = k.expand(B, C, d, h, w).flip(-3, -2, -1).reshape(B * C, 1, d, h, w)
    if pad != "valid":
        pd, ph, pw = d // 2, h // 2, w // 2
        x = F.pad(x, (pw - (w - 1) % 2, pw, ph - (h - 1) % 2, ph, pd - (d - 1) % 2, pd), mode=pad, value=0)
    out = F.conv3d(x.reshape(1, B * C, *x.shape[-3:]), kk, groups=B * C)
    return out.reshape(B, C, *out.shape[-3:])


def run_case(label, shape, fshape, pad, dev, reps, cg_iters=0):
    import deepinv_b200 as dinv

    g = torch.Generator(device=dev).manual_seed(sum(shape) + sum(fshape))
    x = torch.rand(*shape, device=dev, generator=g)
    k = torch.rand(*fshape, device=dev, generator=g)
    k = k / k.sum(dim=(-3, -2, -1), keepdim=True)
    phys = dinv.physics.Blur(filter=k, padding=pad, device=dev)
    with torch.no_grad():
        t_a, y = timed(lambda: phys.A(x), reps)
        t_at, at = timed(lambda: phys.A_adjoint(y), reps)
    B, C = shape[:2]
    d, h, w = fshape[-3:]
    fma = {"A": B * C * y[0, 0].numel() * d * h * w, "At": B * C * y[0, 0].numel() * d * h * w}  # (the same taps, transposed)
    res = {"case": label, "shape": list(shape), "filter": list(fshape), "padding": pad,
           "A_ms": t_a, "At_ms": t_at,
           "A_peak_share": round(fma["A"] / (t_a["median"] * 1e-3) / FP32_FMA_PER_S, 3),
           "At_peak_share": round(fma["At"] / (t_at["median"] * 1e-3) / FP32_FMA_PER_S, 3)}
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        treps = max(1, min(reps, 3))
        with torch.no_grad():
            t_ta, yr = timed(lambda: torch_conv3d(x, k, pad), treps)
        _, vjp = torch.func.vjp(lambda t: torch_conv3d(t, k, pad), x)
        with torch.no_grad():
            t_tat, (atr,) = timed(lambda: vjp(y), treps)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    res.update(torch_A_ms=t_ta, torch_At_ms=t_tat, rel_l2_A=rel(y, yr), rel_l2_At=rel(at, atr))
    if cg_iters:
        with torch.no_grad():
            t_cg, _ = timed(lambda: phys.prox_l2(torch.zeros_like(x), y, 0.5, max_iter=cg_iters, tol=1e-30), 2)
        res[f"cg{cg_iters}_prox_l2_ms"] = t_cg
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("blur3d_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"card": card(), "results": []}
    for label, shape, fshape, pad, cg in (
            ("a 15^3 circular", (4, 1, 64, 256, 256), (1, 1, 15, 15, 15), "circular", 50),
            ("a 15^3 valid", (4, 1, 64, 256, 256), (1, 1, 15, 15, 15), "valid", 0),
            ("a 21x31x31 circular", (4, 1, 64, 256, 256), (1, 1, 21, 31, 31), "circular", 0),
            ("a 21x31x31 valid", (4, 1, 64, 256, 256), (1, 1, 21, 31, 31), "valid", 0),
            ("b per-channel 11x21x21 circular", (1, 3, 32, 256, 256), (1, 3, 11, 21, 21), "circular", 0)):
        r = run_case(label, shape, fshape, pad, dev, args.reps, cg)
        print(json.dumps(r), flush=True)
        out["results"].append(r)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
