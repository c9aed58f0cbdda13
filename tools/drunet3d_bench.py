"""DRUNet(dim=3) forward on the H100: tc32h / tc32 (split-operand wgmma, csrc/conv_tc32.cu with its depth axis) against a torch
nn.Conv3d restatement in strict fp32 (TF32 off), and 10 iterations of PnP-PGD on 3-D single-coil MRI.

    python tools/drunet3d_bench.py [--json out.json]

Times are CUDA-event medians.  TFLOP/s counts 2 FLOP per multiply-add of every convolution of the reference architecture
(nc = 64/128/256/512, nb = 4, in/out 2 channels + the noise map), computed from the shapes below."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def drunet3d_flops(shape, ch=2, nc=(64, 128, 256, 512), nb=4) -> float:
    B, D, H, W = shape
    v = [B * D * H * W / 8 ** i for i in range(4)]
    f = 2 * 27 * ((ch + 1) * nc[0] + nc[0] * ch) * v[0]          # head + tail
    for i in range(4):
        f += (2 if i < 3 else 1) * nb * 2 * 2 * 27 * nc[i] ** 2 * v[i]   # ResBlocks (down and up stages; the body once)
    for i in range(3):
        f += 2 * 2 * 8 * nc[i] * nc[i + 1] * v[i + 1]              # 2x2x2 down + transposed up
    return f


def torch_forward(sd, x, sigma, nb=4):
    """the reference's forward with torch's conv3d (fp32 weights and activations)"""
    B = x.shape[0]
    t = torch.cat([x, torch.full((B, 1, *x.shape[2:]), sigma, device=x.device)], 1)
    c3 = lambda v, k: F.conv3d(v, sd[k], padding=1)
    rb = lambda v, p: v + c3(F.relu(c3(v, p + ".res.0.weight")), p + ".res.2.weight")

    def blocks(v, name, rng):
        for i in rng:
            v = rb(v, f"{name}.{i}")
        return v

    x1 = c3(t, "m_head.weight")
    x2 = F.conv3d(blocks(x1, "m_down1", range(nb)), sd[f"m_down1.{nb}.weight"], stride=2)
    x3 = F.conv3d(blocks(x2, "m_down2", range(nb)), sd[f"m_down2.{nb}.weight"], stride=2)
    x4 = F.conv3d(blocks(x3, "m_down3", range(nb)), sd[f"m_down3.{nb}.weight"], stride=2)
    v = blocks(x4, "m_body", range(nb))
    v = blocks(F.conv_transpose3d(v + x4, sd["m_up3.0.weight"], stride=2), "m_up3", range(1, nb + 1))
    v = blocks(F.conv_transpose3d(v + x3, sd["m_up2.0.weight"], stride=2), "m_up2", range(1, nb + 1))
    v = blocks(F.conv_transpose3d(v + x2, sd["m_up1.0.weight"], stride=2), "m_up1", range(1, nb + 1))
    return c3(v + x1, "m_tail.weight")


def time_ms(fn, reps=5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP

    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    res = {"gpu": power_limit(), "forward": [], "pnp_pgd_mri3d": None}
    print("card, power limit:", res["gpu"])
    torch.manual_seed(0)
    models = {p: dinv.models.DRUNet(in_channels=2, out_channels=2, pretrained=None, dim=3, precision=p).to(dev).eval()
              for p in ("tc32h", "tc32")}
    sd = models["tc32"].state_dict()
    models["tc32h"].load_state_dict(sd)
    for shape in [(1, 64, 256, 256), (4, 32, 128, 128)]:
        x = torch.randn(shape[0], 2, *shape[1:], device=dev)
        flops = drunet3d_flops(shape)
        with torch.no_grad():
            ref = torch_forward(sd, x, 0.05)
            t_torch = time_ms(lambda: torch_forward(sd, x, 0.05), reps=3, warmup=1)
            row = {"shape": shape, "gflop": flops / 1e9, "torch_fp32_ms": t_torch, "torch_fp32_tflops": flops / t_torch / 1e9}
            for p, m in models.items():
                out = m(x, 0.05)
                row[f"{p}_rel_l2_vs_torch_fp32"] = float((out - ref).norm() / ref.norm())
                t = time_ms(lambda: m(x, 0.05))
                row[f"{p}_ms"], row[f"{p}_tflops"] = t, flops / t / 1e9
            del ref, out
        torch.cuda.empty_cache()
        print(json.dumps(row))
        res["forward"].append(row)
    # 10 iterations of PnP-PGD on 3-D single-coil MRI
    D, H, W = 32, 128, 128
    x = torch.randn(1, 2, D, H, W, device=dev)
    mask = (torch.rand(D, H, W, device=dev) > 0.6).float()
    phys = dinv.physics.MRI(mask=mask, img_size=(2, D, H, W), three_d=True, device=dev)
    y = phys.A(x)
    algo = PGD(data_fidelity=L2(), prior=PnP(models["tc32h"]), stepsize=1.0, sigma_denoiser=0.05, max_iter=10, early_stop=False)
    with torch.no_grad():
        t = time_ms(lambda: algo(y, phys), reps=3, warmup=1)
    res["pnp_pgd_mri3d"] = {"shape": (1, 2, D, H, W), "iterations": 10, "ms": t}
    print(json.dumps(res["pnp_pgd_mri3d"]))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
