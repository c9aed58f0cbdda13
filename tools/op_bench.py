#!/usr/bin/env python
"""Per-operator timings at the BASELINE.json config sizes (CUDA events, inputs resident in HBM).
Writes one JSON object per operator; used to fill profiles/ and DESIGN.md's roofline table."""
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import deepinv_b200 as dinv  # noqa: E402

dev = torch.device("cuda:0")
PEAK = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"] if (ROOT / "MEASURED_PEAKS.json").exists() else 6650.0


USE_GRAPH = "--graph" in sys.argv


def t(fn, iters=10, warmup=3, graph=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    if USE_GRAPH if graph is None else graph:  # replay a captured call: device time without the Python / ctypes launch path
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(g):
            fn()
        fn = g.replay
        fn()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def report(name, ms, mb=None, gflop=None):
    d = {"op": name, "ms": round(ms, 4)}
    if mb is not None:
        d.update(algorithmic_MB=round(mb, 1), GBps=round(mb / ms, 1), frac_hbm=round(mb / ms / PEAK, 4))
    if gflop is not None:
        d.update(gflop=round(gflop, 1), TFLOPs=round(gflop / ms, 2))
    print(json.dumps(d), flush=True)


which = [a for a in sys.argv[1:] if not a.startswith("--")] or ["mri", "tomo", "blur", "mcmri"]
g = torch.Generator(device=dev).manual_seed(0)
with torch.no_grad():
    if "mri" in which:
        B, H, W = 64, 256, 256
        x = torch.randn(B, 2, H, W, device=dev, generator=g)
        cols = (torch.rand(B, 1, 1, W, device=dev, generator=g) > 0.75).float().expand(B, 2, H, W).contiguous()
        full = (torch.rand(B, 2, H, W, device=dev, generator=g) > 0.75).float()
        img = B * 2 * H * W * 4 / 1e6
        for tag, m, extra in (("line mask", cols, 0.0), ("full fp32 mask", full, img)):
            p = dinv.physics.MRI(mask=m, img_size=(2, H, W), device=dev)
            y = p.A(x)
            aty = p.A_adjoint(y)
            report(f"MRI.A 64x256^2 [{tag}]", t(lambda: p.A(x), 50), 2 * img + extra)
            report(f"MRI.A_adjoint [{tag}]", t(lambda: p.A_adjoint(y), 50), 2 * img + extra)
            report(f"MRI.A_adjoint_A [{tag}]", t(lambda: p.A_adjoint_A(x), 50), 2 * img + extra)
            report(f"MRI.normal_step [{tag}]", t(lambda: p.normal_step(x, aty, 1.0), 50), 3 * img + extra)
            report(f"MRI.prox_l2 [{tag}]", t(lambda: p.prox_l2(x, y, 1.0), 50), 3 * img + extra)
    if "tomo" in which:
        B, W, A = 32, 512, 180
        p = dinv.physics.Tomography(angles=A, img_width=W, normalize=False, device=dev)
        x = torch.randn(B, 1, W, W, device=dev, generator=g)
        y = p.A(x)
        mb = (B * W * W + B * p.P * A) * 4 / 1e6
        samples = B * A * p.P * p.P
        report("Tomography.A 32x512^2x180", t(lambda: p.A(x), 5, 2), mb, gflop=samples * 14 / 1e9)
        report("Tomography.A_adjoint (exact transpose)", t(lambda: p.A_adjoint(y), 5, 2), mb, gflop=samples * 14 / 1e9)
        report("Tomography.fbp", t(lambda: p.A_dagger(y, fbp=True), 5, 2), mb + 2 * B * p.P * A * 4 / 1e6)
        pb = dinv.physics.Tomography(angles=A, img_width=W, normalize=False, adjoint_via_backprop=False, device=dev)
        report("Tomography.A_adjoint (IRadon)", t(lambda: pb.A_adjoint(y), 5, 2), mb)
        t0 = time.perf_counter()
        pn = dinv.physics.Tomography(angles=A, img_width=W, normalize=True, device=dev)
        torch.cuda.synchronize()
        report("Tomography.__init__ (power iteration norm=%.2f)" % float(pn.operator_norm), (time.perf_counter() - t0) * 1e3)
        xs = x[:4]
        ys = p.A(xs)
        report("Tomography.prox_l2 (CG<=50) batch 4", t(lambda: p.prox_l2(xs, ys, 1.0), 1, 1, graph=False))
    if "blur" in which:
        B, H, W = 32, 1024, 1024
        x = torch.rand(B, 1, H, W, device=dev, generator=g)
        img = B * H * W * 4 / 1e6
        for k in (31, 3):  # 3 x 3: the fewest FMAs per output, where a per-tile fixed cost shows most
            f = torch.rand(1, 1, k, k, device=dev, generator=g)
            f /= f.sum()
            gf = 2 * k * k * B * H * W / 1e9
            for pad in ("circular", "valid", "reflect", "replicate", "constant"):
                p = dinv.physics.Blur(filter=f, padding=pad, device=dev)
                y = p.A(x)
                report(f"Blur.A 32x1024^2 {k}x{k} [{pad}]", t(lambda: p.A(x), 20, 3), 2 * img, gflop=gf)
                report(f"Blur.A_adjoint {k}x{k} [{pad}]", t(lambda: p.A_adjoint(y), 20, 3), 2 * img, gflop=gf)
        f = torch.rand(1, 1, 31, 31, device=dev, generator=g)
        f /= f.sum()
        pf = dinv.physics.BlurFFT(img_size=(1, H, W), filter=f, device=dev)
        y = pf.A(x)
        report("BlurFFT.A 32x1024^2", t(lambda: pf.A(x), 10, 2), 2 * img)
        report("BlurFFT.A_adjoint", t(lambda: pf.A_adjoint(y), 10, 2), 2 * img)
        report("BlurFFT.prox_l2", t(lambda: pf.prox_l2(x, y, 1.0), 10, 2), 5 * img)
        pc = dinv.physics.Blur(filter=f, padding="circular", device=dev)
        xs, ys = x[:4], pc.A(x[:4])
        report("Blur.prox_l2 (CG<=50) batch 4", t(lambda: pc.prox_l2(xs, ys, 1.0), 1, 1, graph=False))
    if "mcmri" in which:
        B, N, H, W = 32, 8, 320, 320
        x = torch.randn(B, 2, H, W, device=dev, generator=g)
        maps = torch.view_as_complex(torch.randn(1, N, H, W, 2, device=dev, generator=g))
        maps = maps / maps.abs().pow(2).sum(1, keepdim=True).sqrt()
        mask = (torch.rand(B, 1, 1, W, device=dev, generator=g) > 0.875).float().expand(B, 2, H, W).contiguous()
        p = dinv.physics.MultiCoilMRI(mask=mask, coil_maps=maps, img_size=(2, H, W), device=dev)
        y = p.A(x)
        mb = (B * 2 * H * W + B * 2 * N * H * W + N * H * W * 2) * 4 / 1e6
        report("MultiCoilMRI.A 32x8x320^2", t(lambda: p.A(x), 10, 2), mb)
        report("MultiCoilMRI.A_adjoint", t(lambda: p.A_adjoint(y), 10, 2), mb)
        report("MultiCoilMRI.A_dagger (CG)", t(lambda: p.A_dagger(y), 1, 1, graph=False))
if "train" in which:  # backward kernels of the fp32 denoiser path (SURVEY §8(f) item 2) + one unfolded training step
    from deepinv_b200 import ops
    from deepinv_b200.optim import L2, PnP
    from deepinv_b200.unfolded import unfolded_builder

    B, C, H, W = 8, 64, 256, 256
    x = torch.randn(B, C, H, W, device=dev, generator=g)
    w = torch.randn(C, C, 3, 3, device=dev, generator=g) / 24
    gout = torch.randn(B, C, H, W, device=dev, generator=g)
    gf = 2 * 9 * C * C * B * H * W / 1e9
    with torch.no_grad():
        report("conv3x3 fp32 forward 8x64x256^2 (64->64)", t(lambda: ops.conv_f32(x, w), 5, 2, graph=False), gflop=gf)
        wt = w.transpose(0, 1).flip(2, 3).contiguous()
        report("conv3x3 fp32 data gradient", t(lambda: ops.conv_f32(gout, wt), 5, 2, graph=False), gflop=gf)
        report("conv3x3 fp32 weight gradient", t(lambda: ops.conv_f32_wgrad(x, None, gout, w.shape), 5, 2, graph=False), gflop=gf)
        report("relu backward 8x64x256^2", t(lambda: ops.relu_bwd(gout, x), 5, 2, graph=False), 3 * x.numel() * 4 / 1e6)
    Bt = 4
    xt = torch.randn(Bt, 2, 256, 256, device=dev, generator=g)
    cols = (torch.rand(Bt, 1, 1, 256, device=dev, generator=g) > 0.75).float().expand(Bt, 2, 256, 256).contiguous()
    p = dinv.physics.MRI(mask=cols, img_size=(2, 256, 256), device=dev)
    with torch.no_grad():
        yt = p.A(xt)
    den = dinv.models.DRUNet(in_channels=2, out_channels=2, pretrained=None, device=dev).train()
    model = unfolded_builder("PGD", params_algo={"stepsize": [1.0, 1.0], "g_param": [0.05, 0.03], "lambda": 1.0},
                             trainable_params=["stepsize", "g_param"], data_fidelity=L2(), prior=PnP(den), max_iter=2).to(dev)

    def step():
        model.zero_grad(set_to_none=True)
        loss = ((model(yt, p) - xt) ** 2).mean()
        loss.backward()

    # 2 unfolded iterations x (forward 277 GFLOP + data gradient 277 + weight gradient 277) per image
    report("unfolded PGD (2 it, DRUNet fp32) training step, batch 4 x 256^2", t(step, 2, 1, graph=False),
           gflop=2 * 3 * 277.4 * Bt)
