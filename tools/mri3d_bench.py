"""Time 3-D MRI (`MRI` / `MultiCoilMRI` with three_d=True) on the GPU and write a markdown report (profiles/mri3d_h100.md).

    python tools/mri3d_bench.py --out profiles/mri3d_h100.md [--reps 20]

Workloads (seeded synthetic data, sizes a 3-D user runs):
  (a) a knee volume shaped like SKM-TEA: (1, 2, 160, 512, 512), 8 coils (radix-5 depth);
  (b) (2, 2, 128, 256, 256), 16 coils (powers of two, 256² slices);
  (c) single coil (4, 2, 64, 256, 256): A, A^T, A^T A, prox_l2, normal_step, each also through the previous single-coil path
      (the separable transform on the 2-D entry with two permute copies), alternated with the new one in this run;
  (d) a 10-iteration CG A_dagger on (b).
Per call: median and range of CUDA-event times over the repetitions after warm-up, algorithmic bytes (x, maps and mask read as
stored, y written; the reverse for A^T) over the median against 3.35 TB/s, and the same call through a torch restatement of the
reference (torch.fft.fftn with the shifts and complex conversions, deepinv/physics/mri.py:254-324) with the relative L2 distance.
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import deepinv_b200 as dinv  # noqa: E402
from deepinv_b200 import _ffi, ops  # noqa: E402
from deepinv_b200.physics.forward import DecomposablePhysics  # noqa: E402

HBM = 3.35e12


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


# ---- torch restatement of the reference (complex conversions + shifted fftn) -----------------------------------------------------
def _c(x):
    return torch.view_as_complex(x.movedim(1, -1).contiguous())


def _r(x):
    return torch.view_as_real(x).movedim(-1, 1)


def _f3(x, inv=False):
    d = (-3, -2, -1)
    f = torch.fft.ifftn if inv else torch.fft.fftn
    return torch.fft.fftshift(f(torch.fft.ifftshift(x, dim=d), dim=d, norm="ortho"), dim=d)


def ref_mc_A(x, mask, maps):
    return mask[:, :, None] * _r(_f3(maps * _c(x)[:, None]))


def ref_mc_At(y, mask, maps):
    return _r((maps.conj() * _f3(_c(mask[:, :, None] * y), True)).sum(1))


def ref_mc_rss(y, mask):  # the RSS volume the drop-in returns (the reference itself raises on 3-D rss)
    return _f3(_c(mask[:, :, None] * y), True).abs().pow(2).sum(1, keepdim=True).sqrt()


def ref_cg(y, mask, maps, iters):
    """CG on A^T A x = A^T y from x = 0 with the restated operators (deepinv/optim/linear/conjugate_gradient.py, tol 0)"""
    b = ref_mc_At(y, mask, maps)
    x = torch.zeros_like(b)
    r = b.clone()
    p = r.clone()
    rs = (r * r).sum()
    for _ in range(iters):
        ap = ref_mc_At(ref_mc_A(p, mask, maps), mask, maps)
        alpha = rs / (p * ap).sum()
        x = x + alpha * p
        r = r - alpha * ap
        rn = (r * r).sum()
        p = r + (rn / rs) * p
        rs = rn
    return x


# single coil (deepinv/physics/forward.py:1080-1252 with V^T = the shifted fftn)
def ref_A(x, m):
    return m * _r(_f3(_c(x)))


def ref_At(y, m):
    return _r(_f3(_c(m * y), True))


def ref_AtA(x, m):
    return _r(_f3(_c(m * m * _r(_f3(_c(x)))), True))


def ref_prox(z, y, m, gamma):
    b = ref_At(y, m) + z / gamma
    return _r(_f3(_c(_r(_f3(_c(b))) / (m * m + 1 / gamma)), True))


# ---- the previous single-coil 3-D path: the separable transform on the 2-D entry with two permute copies ------------------------
def old_transform3(x, inverse):
    B, _, D, H, W = x.shape
    t = x.permute(0, 2, 1, 3, 4).reshape(B * D, 2, H, W)
    t = ops.spectral(t, H, W, fwd=not inverse, inv=inverse)
    t = t.reshape(B, D, 2, H, W).permute(0, 3, 4, 2, 1).reshape(B * H * W, 2, 1, D)
    t = ops.spectral(t, 1, D, fwd=not inverse, inv=inverse)
    return t.reshape(B, H, W, 2, D).permute(0, 3, 4, 1, 2)


class OldMRI3D(DecomposablePhysics):
    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def V_adjoint(self, x):
        return old_transform3(x, False)

    def V(self, x, **kw):
        return old_transform3(x, True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/mri3d_h100.md")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/mri3d_bench.py measures on the GPU; there is none here"
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    name = card()
    lines = [f"# 3-D MRI on {name}", "",
             f"`tools/mri3d_bench.py --reps {args.reps}`, CUDA events, median [min, max] over {args.reps} repetitions after 3 warm-ups. "
             "GB/s = algorithmic bytes (inputs read as stored, output written) / median; % = of 3.35 TB/s. "
             "torch ref = the reference's arithmetic restated in torch on the same GPU (`torch.fft.fftn` with shifts and complex "
             "conversions); rel L2 = distance between the two outputs.", "",
             "| workload | call | ms median [min, max] | GB/s | % HBM | torch ref ms | rel L2 |", "|---|---|---|---|---|---|---|"]

    def row(wl, call, t, nbytes, tref=None, err=None):
        gbs = nbytes / (t[0] * 1e-3) / 1e9
        r = f"{tref[0]:.3f}" if tref else "-"
        e = f"{err:.2e}" if err is not None else "-"
        lines.append(f"| {wl} | {call} | {t[0]:.3f} [{t[1]:.3f}, {t[2]:.3f}] | {gbs:.0f} | {100 * gbs * 1e9 / HBM:.0f} | {r} | {e} |")
        print(lines[-1], flush=True)

    g = torch.Generator(device=dev).manual_seed(0)
    # ---- (a), (b): multi-coil --------------------------------------------------------------------------------------------------
    for wl, (B, D, H, W, N) in (("(a) 1x160x512x512, 8 coils", (1, 160, 512, 512, 8)), ("(b) 2x128x256x256, 16 coils", (2, 128, 256, 256, 16))):
        V = D * H * W
        x = torch.randn(B, 2, D, H, W, device=dev, generator=g)
        maps = torch.randn(1, N, D, H, W, device=dev, generator=g, dtype=torch.complex64)
        maps = maps / maps.abs().pow(2).sum(1, keepdim=True).sqrt()
        mask = (torch.rand(D, H, W, device=dev, generator=g) > 0.7).float()
        phys = dinv.physics.MultiCoilMRI(mask=mask, coil_maps=maps, img_size=(2, D, H, W), three_d=True, device=dev)
        m5 = phys.mask
        with torch.no_grad():
            y = phys.A(x)
            t = timed(lambda: phys.A(x), args.reps)
            yr = ref_mc_A(x, m5, maps)
            tr = timed(lambda: ref_mc_A(x, m5, maps), max(3, args.reps // 4))
            row(wl, "A", t, 4 * (2 * B * V + 2 * N * V + 2 * V + 2 * B * N * V), tr, rel(y, yr))
            del yr
            at = phys.A_adjoint(y)
            t = timed(lambda: phys.A_adjoint(y), args.reps)
            ar = ref_mc_At(y, m5, maps)
            tr = timed(lambda: ref_mc_At(y, m5, maps), max(3, args.reps // 4))
            row(wl, "A^T", t, 4 * (2 * B * N * V + 2 * N * V + 2 * V + 2 * B * V), tr, rel(at, ar))
            del ar
            t = timed(lambda: phys.A_adjoint(y, rss=True), args.reps)
            tr = timed(lambda: ref_mc_rss(y, m5), max(3, args.reps // 4))
            row(wl, "A^T rss", t, 4 * (2 * B * N * V + 2 * V + B * V), tr, rel(phys.A_adjoint(y, rss=True), ref_mc_rss(y, m5)))
            if wl.startswith("(b)"):
                phys.max_iter, phys.tol = 10, 0.0
                t = timed(lambda: phys.A_dagger(y), max(3, args.reps // 4), warm=1)
                tr = timed(lambda: ref_cg(y, m5, maps, 10), 3, warm=1)
                row("(d) CG A_dagger on (b), 10 iterations", "A_dagger", t, 10 * 4 * 2 * (2 * B * V + 2 * N * V + 2 * V + 2 * B * N * V),
                    tr, rel(phys.A_dagger(y), ref_cg(y, m5, maps, 10)))
        ws = ops._ws_cache.get((dev, "spectral"))
        lines.append(f"| {wl} | workspace | {ws.numel() / 2**30:.2f} GiB (`dinvk_spectral3d_workspace_bytes`) | | | | |")
        del x, maps, phys, y, at
        ops._ws_cache.clear()
        torch.cuda.empty_cache()
    # ---- (c): single coil, new path vs the previous one, alternated ------------------------------------------------------------
    B, D, H, W = 4, 64, 256, 256
    V = D * H * W
    x = torch.randn(B, 2, D, H, W, device=dev, generator=g)
    z = torch.randn(B, 2, D, H, W, device=dev, generator=g)
    mask = (torch.rand(D, H, W, device=dev, generator=g) > 0.7).float()
    new = dinv.physics.MRI(mask=mask, img_size=(2, D, H, W), three_d=True, device=dev)
    old = OldMRI3D(new.mask)
    wl = "(c) 4x64x256x256, single coil"
    with torch.no_grad():
        y = new.A(x)
        aty = new.A_adjoint(y)
        m = new.mask
        calls = {"A": (lambda p: p.A(x), 4 * (2 * B * V + 2 * V + 2 * B * V), lambda: ref_A(x, m)),
                 "A^T": (lambda p: p.A_adjoint(y), 4 * (2 * B * V + 2 * V + 2 * B * V), lambda: ref_At(y, m)),
                 "A^T A": (lambda p: p.A_adjoint_A(x), 4 * (2 * B * V + 2 * V + 2 * B * V), lambda: ref_AtA(x, m)),
                 "prox_l2": (lambda p: p.prox_l2(z, y, 0.5) if p is new else DecomposablePhysics.prox_l2(p, z, y, 0.5),
                             4 * (2 * 2 * B * V + 2 * V + 2 * B * V), lambda: ref_prox(z, y, m, 0.5)),
                 "normal_step": (lambda p: p.normal_step(x, aty, 0.5) if p is new else x - 0.5 * (p.A_adjoint_A(x) - aty),
                                 4 * (3 * 2 * B * V + 2 * V + 2 * B * V), lambda: x - 0.5 * (ref_AtA(x, m) - aty))}
        regress = []
        for cname, (fn, nbytes, reff) in calls.items():
            tn, to = [], []
            for _ in range(3):  # alternate the two paths
                tn.append(timed(lambda: fn(new), args.reps))
                to.append(timed(lambda: fn(old), args.reps))
            best = lambda ts: sorted(ts)[1]  # noqa: E731  (median of the three medians)
            d = rel(fn(new), fn(old))
            row(wl, cname, best(tn), nbytes, timed(reff, args.reps), rel(fn(new), reff()))
            regress.append(f"| {cname} | {best(tn)[0]:.3f} | {best(to)[0]:.3f} | {best(to)[0] / best(tn)[0]:.2f}x | {d:.1e} |")
    lines += ["", f"Single coil (c): the fused 3-D entry against the previous path (the separable transform on the 2-D entry, two "
              "permute copies per transform, generic SVD bodies), alternated three times in this run; ms = median of the three medians.",
              "", "| call | new ms | previous ms | speed-up | rel L2 new vs previous |", "|---|---|---|---|---|", *regress]
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
