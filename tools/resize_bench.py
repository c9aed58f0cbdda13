"""Time the MATLAB-bicubic resize (libdinvk `dinvk_resize_fwd` / `dinvk_resize_adj`: `DownsamplingMatlab.A` / `A_adjoint`) on
the GPU.

Workloads, seeded inputs at super-resolution sizes: (64, 3, 256, 256) at factor 4 and (8, 3, 1080, 1920) at factor 2.
For A and A^T: ms per eager call (CUDA events, median and range of --reps after a warm-up; host Python included), the kernel
time per call (20 calls replayed from one CUDA graph), the HBM bytes the kernel must move (input read once, output written once,
from the shapes) over the kernel time as a fraction of the 3.35 TB/s data-sheet bound, and, in the same run, a torch
restatement of the reference's algorithm (imresize.py resize_1d: reflect padding by index, unfold, gather, multiply, sum over
the taps, H then W) and its autograd adjoint, with the relative L2 distance between the two.  Card name and
power limit are read in the same run.

    python tools/resize_bench.py [--reps N] [--out FILE]

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


def graph_timed(fn, reps: int, calls: int = 20) -> dict:
    """kernel time per call: `calls` calls captured in one CUDA graph and replayed, so the host's Python cost per call (larger
    than these kernels at these sizes) does not starve the GPU"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    t, _ = timed(lambda: g.replay(), reps)
    return {k: round(v / calls, 4) for k, v in t.items()}


def torch_resize_1d(x, dim, tab):
    """one resize_1d pass restated with torch ops: reflect-pad by an index map, unfold k taps, pick every output's window,
    multiply by its weights and sum over the taps (x: (N, 1, H, W))"""
    n = x.shape[dim]
    k = tab.k
    base = tab.base.long().to(x.device)
    lo = -int(base.min().clamp(max=0))
    hi = max(0, int(base.max()) + k - n)
    j = torch.arange(-lo, n + hi, device=x.device)
    j = torch.where(j < 0, -1 - j, torch.where(j >= n, 2 * n - 1 - j, j))
    xp = x.index_select(dim, j)
    w = tab.weight.t().to(x.device)  # (k, n_out)
    if dim == 2:
        u = F.unfold(xp, (k, 1)).view(x.shape[0], k, xp.shape[2] - k + 1, x.shape[3])
        return (u[:, :, base + lo, :] * w.view(1, k, -1, 1)).sum(1, keepdim=True)
    u = F.unfold(xp, (1, k)).view(x.shape[0], k, x.shape[2], xp.shape[3] - k + 1)
    return (u[..., base + lo] * w.view(1, k, 1, -1)).sum(1, keepdim=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "resize_bench needs a CUDA device"
    import deepinv_b200 as dinv
    from deepinv_b200.physics.imresize import resize_plan

    res = {"card": card(), "workloads": []}
    for shape, f in (((64, 3, 256, 256), 4), ((8, 3, 1080, 1920), 2)):
        B, C, H, W = shape
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.rand(shape, device="cuda", generator=g)
        p = dinv.physics.DownsamplingMatlab(factor=f, device="cuda")
        (Ho, Wo), th, tw = resize_plan(H, W, scale=1 / f)
        v = torch.randn(B, C, Ho, Wo, device="cuda", generator=g)
        with torch.no_grad():
            t_a, y = timed(lambda: p.A(x), a.reps)
            t_at, xt = timed(lambda: p.A_adjoint(v), a.reps)
            k_a, k_at = graph_timed(lambda: p.A(x), a.reps), graph_timed(lambda: p.A_adjoint(v), a.reps)
        nbytes = 4 * B * C * (H * W + Ho * Wo)
        bound_ms = nbytes / HBM_BYTES_PER_S * 1e3

        def ref_A(t):
            t = t.reshape(-1, 1, H, W)
            return torch_resize_1d(torch_resize_1d(t, 2, th), 3, tw).reshape(B, C, Ho, Wo)

        with torch.no_grad():
            t_ref, y_ref = timed(lambda: ref_A(x), max(5, a.reps // 5))
        xg = torch.zeros_like(x, requires_grad=True)

        def ref_At():
            (gx,) = torch.autograd.grad(ref_A(xg), xg, v)
            return gx

        t_ref_t, xt_ref = timed(ref_At, max(5, a.reps // 5))
        rel = lambda u, w: float((u.double() - w.double()).norm() / w.double().norm())  # noqa: E731
        res["workloads"].append({
            "shape": list(shape), "factor": f, "out": [Ho, Wo], "taps": [th.k, tw.k], "bytes": nbytes,
            "hbm_bound_ms": round(bound_ms, 4),
            "A_call_ms": t_a, "At_call_ms": t_at,
            "A_kernel_ms": k_a, "A_hbm_fraction": round(bound_ms / k_a["median"], 3),
            "At_kernel_ms": k_at, "At_hbm_fraction": round(bound_ms / k_at["median"], 3),
            "torch_restatement_A_ms": t_ref, "torch_restatement_autograd_At_ms": t_ref_t,
            "rel_A_vs_restatement": rel(y, y_ref), "rel_At_vs_restatement": rel(xt, xt_ref),
            "speedup_A_per_call": round(t_ref["median"] / t_a["median"], 1),
            "speedup_At_per_call": round(t_ref_t["median"] / t_at["median"], 1),
        })
        del x, v, y, xt, y_ref, xt_ref, xg
        torch.cuda.empty_cache()
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
