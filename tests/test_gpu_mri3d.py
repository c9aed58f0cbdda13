"""3-D MRI on the GPU: every launch path of `dinvk_spectral3d` against the fp64 restatement (tests/mri3d_path_cases.py, with a
per-row kernel census under torch.profiler), the refused shapes, a coil tensor past 2^31 floats, and `MRI(three_d=True)` /
`MultiCoilMRI(three_d=True)` through the package API against the mri3d_* golden vectors of the reference (A, A^T, crop, CG SENSE
A_dagger, prox_l2, PGD with L2 + Tikhonov), with the reference's recorded rss / mag errors replaced by the true RSS volume."""
import json
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import mri3d_path_cases as T  # noqa: E402
import mri3d_ref64 as S  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")  # the fixtures' err_* codes (make_golden_mri3d.py)
MC_CASES = [n for n in golden_names("mri3d_mc_") if n != "mri3d_mc_pgd"]
SC_CASES = golden_names("mri3d_sc_")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row, dev):
    res = T.check_row(row, dev)
    print(f"\n{row.name}: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in res.items()))


def test_einval(dev):
    from deepinv_b200 import ops

    for name, rc, msg in T.run_einval(ops.get_lib(), dev):
        assert rc == 1, (name, rc, msg)
        assert msg, name


def test_coil_tensor_past_2_31_floats(dev):
    """260 coils of 64 x 256 x 256: y holds 2.18e9 floats, so its last coils sit past 2^31 from the start.  The forward is checked
    coil by coil on the last coils against fp64 on the CPU; the adjoint against an fp64 evaluation of the contract on the GPU."""
    from deepinv_b200 import ops

    N, D, H, W = 260, 64, 256, 256
    assert 2 * N * D * H * W > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.randn(1, 2, D, H, W, device=dev, generator=g)
    maps = torch.randn(1, N, D, H, W, device=dev, generator=g, dtype=torch.complex64)
    mask = (torch.rand(1, 2, D, H, W, device=dev, generator=g) > 0.5).float()
    spec = ops.mask_spec3d(mask)
    y = ops.spectral3d(x, D, H, W, fwd=True, inv=False, gmode=1, mask=spec, ncoil=N, coil_mode=1, coil_maps=maps)
    torch.cuda.synchronize()
    xc = torch.complex(x[:, 0].double(), x[:, 1].double()).cpu()
    m = mask.double().cpu()
    for n in (0, N - 2, N - 1):
        want = S.fft3(maps[:, n].cpu().to(torch.complex128) * xc, False)
        want = torch.stack([want.real * m[:, 0], want.imag * m[:, 1]], 1)
        assert rel_err(y[:, :, n], want) < TOL, n
    at = ops.spectral3d(y, D, H, W, fwd=False, inv=True, gmode=1, mask=spec, ncoil=N, coil_mode=2, coil_maps=maps)
    acc = torch.zeros(1, D, H, W, dtype=torch.complex128, device=dev)
    md = mask.double()
    for n0 in range(0, N, 20):
        yc = y[:, :, n0:n0 + 20].double()
        u = torch.complex(yc[:, 0] * md[:, 0, None], yc[:, 1] * md[:, 1, None])
        v = S.fft3(u, True)
        acc += (maps[:, n0:n0 + 20].to(torch.complex128).conj() * v).sum(1)
    want = torch.stack([acc.real, acc.imag], 1)
    assert rel_err(at, want) < TOL


def test_kernel_census(dev):
    """every table row launched exactly its kernels, and the physics methods launch the library's kernels only (no cuFFT, no
    permute or copy kernel).  The profiler runs in a child process, so the pytest process's tracer is left alone."""
    code = f"import sys; sys.path.insert(0, {str(HERE)!r}); import test_gpu_mri3d as G; G._census_child()"
    p = subprocess.run([sys.executable, "-c", code], cwd=str(HERE.parent), capture_output=True, text=True, timeout=1200)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("CENSUS_JSON ")]
    assert p.returncode == 0 and lines, f"child failed ({p.returncode}):\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    rep = json.loads(lines[-1][len("CENSUS_JSON "):])
    if rep["no_cupti"]:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable); the numeric tests do not depend on it")
    assert not rep["wrong"], f"rows that did not launch exactly their kernels: {rep['wrong']}"
    assert not rep["physics"], f"physics methods that launched other kernels: {rep['physics']}"
    assert all(any(k in n for n in rep["seen"]) for k in T.LIBRARY_KERNELS)


def _census_child():
    from torch.profiler import ProfilerActivity, profile

    import deepinv_b200 as dinv

    dev = torch.device("cuda:0")

    def kernels(fn):
        for _ in range(10):  # the tracer now and then delivers no record at all for a profile: no evidence, retry
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names = {re.sub(r"\s+", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
            if names:
                return names
        return set()

    probe = torch.ones(1024, device=dev)
    if not kernels(lambda: probe.mul_(2)):
        print("CENSUS_JSON " + json.dumps({"no_cupti": True}))
        return
    seen, wrong = set(), []
    for row in T.ROWS:
        if not row.kernels:
            continue
        call = T.Case(row, dev).make_call()
        call()  # first use of a size uploads its twiddle tables (a host-to-device copy): not part of the census
        names = kernels(call)
        seen |= names
        miss = [k for k in row.kernels if not any(k in n for n in names)]
        extra = [n for n in names if not any(k in n for k in row.kernels)]
        if miss or extra:
            wrong.append((row.name, miss, extra))
    # the physics classes: nothing but library kernels for the operator bodies
    g = torch.Generator().manual_seed(0)
    dims = (32, 48, 64)
    x = torch.randn(2, 2, *dims, generator=g).to(dev)
    maps = torch.randn(1, 4, *dims, generator=g, dtype=torch.complex64).to(dev)
    mask = (torch.rand(*dims, generator=g) > 0.5).float().to(dev)
    mc = dinv.physics.MultiCoilMRI(mask=mask, coil_maps=maps, img_size=(2, *dims), three_d=True, device=dev)
    sc = dinv.physics.MRI(mask=mask, img_size=(2, *dims), three_d=True, device=dev)
    y, ys = mc.A(x), sc.A(x)
    aty = sc.A_adjoint(ys)
    calls = {"mc A": lambda: mc.A(x), "mc At": lambda: mc.A_adjoint(y), "mc rss": lambda: mc.A_adjoint(y, rss=True),
             "sc A": lambda: sc.A(x), "sc At": lambda: sc.A_adjoint(ys), "sc AtA": lambda: sc.A_adjoint_A(x),
             "sc prox": lambda: sc.prox_l2(x, ys, 0.5), "sc dagger": lambda: sc.A_dagger(ys),
             "sc normal_step": lambda: sc.normal_step(x, aty, 0.5), "sc V": lambda: sc.V(x), "sc Vt": lambda: sc.V_adjoint(x)}
    physics = []
    with torch.no_grad():
        for name, fn in calls.items():
            fn()
            names = kernels(fn)
            other = [n for n in names if not any(k in n for k in T.LIBRARY_KERNELS)]
            if other or not names:
                physics.append((name, other))
    print("CENSUS_JSON " + json.dumps({"no_cupti": False, "wrong": wrong, "seen": sorted(seen), "physics": physics}))


def _maps(g, dev):
    return torch.complex(g["maps_re"], g["maps_im"]).to(dev)


@pytest.mark.parametrize("name", MC_CASES)
def test_multicoil_golden(name, dev):
    import deepinv_b200 as dinv

    g = load_golden(name)
    x, y = g["x"].to(dev), g["y"].to(dev)
    phys = dinv.physics.MultiCoilMRI(mask=g["mask_in"].to(dev), coil_maps=_maps(g, dev), img_size=tuple(x.shape[1:]), three_d=True,
                                     device=dev)
    assert torch.equal(phys.mask.cpu(), g["mask"])
    phys.max_iter, phys.tol = int(g["max_iter"]), float(g["tol"])
    with torch.no_grad():
        yk = phys.A(x)
        assert rel_err(yk, g["y"]) < TOL and torch.equal((yk == 0).cpu(), g["y"] == 0)
        assert rel_err(phys.A_adjoint(y), g["At"]) < TOL
        assert rel_err(phys.A_adjoint(y, crop=True), g["At_crop"]) < TOL
        # the reference raises here (err_rss); the drop-in returns the RSS volume, pinned by the fp64 restatement
        rss = phys.A_adjoint(y, rss=True)
        want = S.mc_At(g["y"].double(), g["mask"].double(), torch.complex(g["maps_re"], g["maps_im"]), rss=True)
        assert int(g["err_rss"]) == ERRORS.index("ValueError") and rss.shape == want.shape and rel_err(rss, want) < TOL
        assert rel_err(phys.A_dagger(y), g["dagger"]) < 1e-4
        assert rel_err(phys.prox_l2(g["z"].to(dev), y, float(g["gamma"])), g["prox"]) < 1e-4
    # mask= / coil_maps= given to a method are stored, as in 2-D
    m2 = torch.ones_like(g["mask_in"]).to(dev)
    phys.A(x, mask=m2)
    assert torch.equal(phys.mask, phys.check_mask(m2, three_d=True))
    # autograd through linear_apply: the gradient of <A x, v> is A^T v
    xr = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad((phys.A(xr) * y).sum(), xr)
    assert rel_err(gx, phys.A_adjoint(y)) < 1e-6


@pytest.mark.parametrize("name", SC_CASES)
def test_single_coil_golden(name, dev):
    import deepinv_b200 as dinv

    g = load_golden(name)
    x, y, z = g["x"].to(dev), g["y"].to(dev), g["z"].to(dev)
    phys = dinv.physics.MRI(mask=g["mask_in"].to(dev), img_size=tuple(x.shape[1:]), three_d=True, device=dev)
    gamma = float(g["gamma"])
    with torch.no_grad():
        yk = phys.A(x)
        assert rel_err(yk, g["y"]) < TOL and torch.equal((yk == 0).cpu(), g["y"] == 0)
        aty = phys.A_adjoint(y)
        assert rel_err(aty, g["At"]) < TOL
        assert rel_err(phys.A_adjoint_A(x), g["AtA"]) < TOL
        assert rel_err(phys.A_dagger(y), g["dagger"]) < TOL
        assert rel_err(phys.prox_l2(z, y, gamma), g["prox"]) < TOL
        assert rel_err(phys.prox_l2(z, y, gamma), g["prox"]) < TOL  # the cached A^T y
        gb = torch.full((x.shape[0],), gamma, device=dev)
        assert rel_err(phys.prox_l2(z, y, gb), g["prox"]) < TOL  # per-sample gamma
        step = phys.normal_step(x, aty, 0.3)
        assert rel_err(step, x.cpu() - 0.3 * (g["AtA"] - g["At"])) < TOL
        assert rel_err(phys.A_A_adjoint(y), phys.A(phys.A_adjoint(y))) < TOL
        assert rel_err(phys.V(phys.V_adjoint(x)), x) < TOL
        # the reference raises here (err_mag); the drop-in returns |A^T y|
        mag = phys.A_adjoint(y, mag=True)
        assert int(g["err_mag"]) == ERRORS.index("ValueError") and rel_err(mag, g["At"].pow(2).sum(1, keepdim=True).sqrt()) < TOL


def test_pgd_multicoil(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("mri3d_mc_pgd")
    phys = dinv.physics.MultiCoilMRI(mask=g["mask"].to(dev), coil_maps=_maps(g, dev), img_size=tuple(g["x"].shape[1:]),
                                     three_d=True, device=dev)
    with torch.no_grad():
        out = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=8, early_stop=False)(g["y"].to(dev), phys)
    assert rel_err(out, g["pgd"]) < TOL


def test_transform_of_a_coil_stack(dev):
    """V / V^T of the mixin on a (B,2,N,D,H,W) k-space transform every coil volume (the reference's fftn over (-3,-2,-1))"""
    import deepinv_b200 as dinv

    g = torch.Generator().manual_seed(5)
    y = torch.randn(2, 2, 3, 8, 16, 64, generator=g)
    mix = dinv.physics.mri.MRIMixin()
    for inverse, fn in ((False, mix.im_to_kspace), (True, mix.kspace_to_im)):
        want = S.fft3(torch.complex(y[:, 0].double(), y[:, 1].double()), inverse)
        assert rel_err(fn(y.to(dev), three_d=True), torch.stack([want.real, want.imag], 1)) < TOL
    with pytest.raises(ValueError):
        mix.im_to_kspace(torch.randn(2, 2, 16, 64, device=dev), three_d=True)


def test_shape_errors(dev):
    import deepinv_b200 as dinv

    dims = (4, 6, 8)
    maps = torch.ones(2, 3, *dims, dtype=torch.complex64, device=dev)
    phys = dinv.physics.MultiCoilMRI(coil_maps=maps, img_size=(2, *dims), three_d=True, device=dev)
    with pytest.raises(ValueError):
        phys.A(torch.randn(3, 2, *dims, device=dev))  # coil-map batch 2 against input batch 3
    with pytest.raises(ValueError):
        phys.A(torch.randn(2, 2, 4, 6, 9, device=dev))  # volume size
    sc = dinv.physics.MRI(img_size=(2, *dims), three_d=True, device=dev)
    with pytest.raises(ValueError):
        sc.A(torch.randn(1, 2, 6, 8, device=dev))
