"""Time the TGV prox (libdinvk `dinvk_tgv_prox`) on the GPU.

Workloads
  (a) one TGVDenoiser prox, 1000 iterations, crit = 0 (no early stop), at (64, 2, 256, 256) and (32, 1, 1024, 1024);
  (b) PGD with PnP(TGVDenoiser()) (defaults: crit 1e-5, at most 1000 inner iterations) on the cfg2 MRI problem
      (64, 2, 256, 256), 5 outer iterations.
Prints the card and its power limit, ms per prox, TGV iterations per second, libdinvk launches and host synchronisations
per prox, the algorithmic HBM bytes per launch and the share of the bound derived from shapes, and the same prox run by
the torch restatement (tests/tgv_oracle.py) on the same GPU with the relative L2 distance between the two outputs.

    python tools/tgv_bench.py [--quick] [--lib path/to/libdinvk.so] [--no-oracle]

`--lib` loads another build of the library (e.g. one compiled with -DDINVK_TGV_TILE=.. -DDINVK_TGV_BLOCK=..) for a
(T, K) sweep.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

import torch  # noqa: E402

from tv_bench import FP32_FLOPS, HBM_BYTES_PER_S, card, image  # noqa: E402

# tmp 10, x 8, v 2, x2 relaxation 3, r 11, w 4, r2 relaxation 6, d 4, epsilon 4, dual step 8, norm 9, projection 4,
# u2 relaxation 12
FLOP_PER_PIXEL_IT = 85
BYTES_PER_PIXEL = 60  # read y, x2, r2 (2 floats), u2 (4 floats) = 32 B; write x2, r2, u2 = 28 B


def prox_run(shape, dev, reps, oracle):
    from deepinv_b200 import launch_count, ops
    import tgv_oracle as O

    T, K = ops.tgv_block()
    y = image(shape, 0, dev)
    lam = torch.full((shape[0],), 0.1, device=dev)
    tl1, l2 = 0.01 * (lam * 0.1), lam * 0.15
    r0, u0 = torch.zeros(*shape, 2, device=dev), torch.zeros(*shape, 4, device=dev)
    ops.tgv_prox(y, tl1, l2, y, r0, u0, n_it_max=2 * K, crit=0.0)  # warm-up
    torch.cuda.synchronize()
    times, stats = [], {}
    for _ in range(reps):
        n0 = launch_count()
        t0 = time.perf_counter()
        x, _, _, n = ops.tgv_prox(y, tl1, l2, y, r0, u0, n_it_max=1000, crit=0.0, stats=stats)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        launches = launch_count() - n0
    ms = sorted(times)[len(times) // 2] * 1e3
    npx = y.numel()
    launch_ms = ms / max(stats["launches"], 1)
    bytes_launch = BYTES_PER_PIXEL * npx
    t_hbm = bytes_launch / HBM_BYTES_PER_S * 1e3
    t_fp32 = FLOP_PER_PIXEL_IT * K * npx / FP32_FLOPS * 1e3
    bound = "HBM" if t_hbm >= t_fp32 else "FP32"
    r = {"shape": list(shape), "tile_T": T, "iters_per_launch_K": K, "iterations": int(n), "ms_per_prox": round(ms, 3),
         "ms_all": [round(t * 1e3, 3) for t in times], "tgv_it_per_s": round(1000 / (ms / 1e3), 1),
         "libdinvk_launches_per_prox": int(launches), "tgv_cp_launches": stats["launches"], "host_syncs_per_prox": stats["syncs"],
         "hbm_bytes_per_launch": bytes_launch, "halo_fraction": round((T + 4 * K) ** 2 / T ** 2, 3),
         "hbm_ms_per_launch": round(t_hbm, 4), "fp32_ms_per_launch": round(t_fp32, 4),
         "bound": bound, "bound_ms_per_launch": round(max(t_hbm, t_fp32), 4), "ms_per_launch": round(launch_ms, 4),
         "share_of_bound": round(max(t_hbm, t_fp32) / launch_ms, 3)}
    if oracle:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xr, _, _, nr, _ = O.tgv_denoise(y, 0.1, n_it_max=1000, crit=0.0)
        torch.cuda.synchronize()
        r["oracle_torch_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        r["oracle_iterations"] = nr
        r["rel_l2_vs_oracle"] = float((x.double() - xr.double()).norm() / xr.double().norm())
        r["speedup_vs_oracle"] = round(r["oracle_torch_ms"] / ms, 1)
    return r


def pgd_run(dev, reps):
    import deepinv_b200 as dinv
    from deepinv_b200 import launch_count
    from deepinv_b200.optim import L2, PGD, PnP

    B, H, W = 64, 256, 256
    g = torch.Generator().manual_seed(0)
    x = image((B, 2, H, W), 1, torch.device("cpu"))
    cols = (torch.rand(B, 1, 1, W, generator=g) > 0.7).float()
    cols[..., W // 2 - 8: W // 2 + 8] = 1
    mask = cols.expand(B, 2, H, W).contiguous().to(dev)
    phys = dinv.physics.MRI(mask=mask, img_size=(2, H, W), device=dev)
    y = phys.A(x.to(dev))
    out = []
    for _ in range(reps):
        den = dinv.models.TGVDenoiser()
        algo = PGD(data_fidelity=L2(), prior=PnP(den), stepsize=1.0, sigma_denoiser=0.05, max_iter=5, early_stop=False)
        torch.cuda.synchronize()
        n0 = launch_count()
        t0 = time.perf_counter()
        with torch.no_grad():
            algo(y, phys)
        torch.cuda.synchronize()
        out.append({"s": round(time.perf_counter() - t0, 3), "launches": launch_count() - n0,
                    "last_prox_iterations": int(den.n_iter)})
    return {"workload": "PGD + PnP(TGVDenoiser()) on cfg2 MRI (64, 2, 256, 256), 5 outer iterations, sigma 0.05", "runs": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="one shape, one repetition, no PGD")
    ap.add_argument("--lib", default=None, help="load this libdinvk.so instead of the package's")
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tgv_bench.py needs a CUDA device")
    if a.lib:
        from deepinv_b200 import _lib

        _lib._LIB_PATH = Path(a.lib).resolve()
    dev = torch.device("cuda:0")
    res = {"card": card(), "prox": []}
    print(json.dumps(res["card"]), flush=True)
    shapes = [(64, 2, 256, 256)] if a.quick else [(64, 2, 256, 256), (32, 1, 1024, 1024)]
    for s in shapes:
        res["prox"].append(prox_run(s, dev, 1 if a.quick else a.reps, not a.no_oracle))
        print(json.dumps(res["prox"][-1]), flush=True)
    if not a.quick:
        res["pgd"] = pgd_run(dev, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
