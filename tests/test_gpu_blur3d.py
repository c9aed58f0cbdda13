"""3-D Blur on the GPU: every launch path of `blur3d_corr_kernel` / `blur3d_fold_kernel` against the fp64 restatement
(tests/blur3d_path_cases.py, with a per-row kernel census under torch.profiler), the `blur3d_*` golden vectors of the reference
through the package API at 1e-5, the reference's error types, the rank dispatch of `Blur`, autograd through the opposite kernel,
and CG `prox_l2`, PGD with Tikhonov and GD with ZeroPrior on a 3-D circular blur."""
import json
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import blur3d_path_cases as T  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
OPERATOR_CASES = [n for n in golden_names("blur3d_") if n != "blur3d_algo"]
PADS = T.PADS


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row, dev):
    res = T.check_row(row, dev)
    print(f"\n{row.name}: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in res.items()))


def test_kernel_census(dev):
    """every row launched exactly the kernels it names, and the table as a whole reaches both.  The profiler runs in a child
    process, so this file never starts the tracer of the pytest process: after its first session the tracer now and then
    delivers an empty trace, and tests/test_gpu_blur_paths.py (which sorts after this file) probes it once, without a retry,
    and skips on an empty trace.  Its probe stays the first session of the process."""
    code = f"import sys; sys.path.insert(0, {str(HERE)!r}); import test_gpu_blur3d as G; G._census_child()"
    p = subprocess.run([sys.executable, "-c", code], cwd=str(HERE.parent), capture_output=True, text=True, timeout=1200)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("CENSUS_JSON ")]
    assert p.returncode == 0 and lines, f"child failed ({p.returncode}):\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    rep = json.loads(lines[-1][len("CENSUS_JSON "):])
    if rep["no_cupti"]:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable); the numeric tests do not depend on it")
    assert not rep["wrong"], f"rows that did not launch exactly their kernels: {rep['wrong']}"
    assert all(any(k in n for n in rep["seen"]) for k in (T.K_CORR, T.K_FOLD))


def _census_child():
    """the census of test_kernel_census, in its own process; prints one CENSUS_JSON line"""
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return {re.sub(r"\s+", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}

    probe = torch.ones(1024, device=dev)
    if not kernels(lambda: probe.mul_(2)):  # (the first profile also initialises the tracer)
        print("CENSUS_JSON " + json.dumps({"no_cupti": True}))
        return
    seen, wrong = set(), []
    for row in T.ROWS:
        if row.error or not row.kernels or row.gpu_only:
            continue
        case = T.Case(row, dev)
        with T._env(row.env):
            call = case.make_call()
            for _ in range(10):  # the tracer now and then delivers no record at all for a profile (three in a row seen): no evidence, retry
                names = kernels(call)
                if names:
                    break
        seen |= names
        miss = [k for k in row.kernels if not any(k in n for n in names)]
        extra = [n for n in names if "blur" in n and not any(k in n for k in row.kernels)]
        if miss or extra:
            wrong.append((row.name, miss, extra, sorted(names)))
    print("CENSUS_JSON " + json.dumps({"no_cupti": False, "wrong": wrong, "seen": sorted(seen)}))


def _fold_defect(pad, fs):
    """the reference's transpose is not the transpose there (tests/test_blur3d_ref64.py); ours is pinned by the table"""
    return (pad == "circular" and min(fs) <= 2) or (pad in ("replicate", "reflect") and min(fs) == 1)


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name, dev):
    import deepinv_b200 as dinv

    g = load_golden(name)
    x, k = g["x"].to(dev), g["k"].to(dev)
    fs = tuple(k.shape[-3:])
    for pad in PADS:
        phys = dinv.physics.Blur(filter=k, padding=pad, use_fft=bool(int(g["use_fft"])), device=dev)
        if f"err_{pad}" in g:
            if _fold_defect(pad, fs):
                continue
            with pytest.raises(RuntimeError):  # the reference's type (DinvkError is a RuntimeError)
                phys.A(x)
            continue
        assert rel_err(phys.A(x), g[f"A_{pad}"]) < TOL, (name, pad)
        if not _fold_defect(pad, fs):
            assert rel_err(phys.A_adjoint(g[f"v_{pad}"].to(dev)), g[f"At_{pad}"]) < TOL, (name, pad)


def test_rank_dispatch_and_errors(dev):
    import deepinv_b200 as dinv

    k3 = torch.rand(1, 1, 3, 3, 3, device=dev)
    x = torch.rand(2, 1, 6, 8, 8, device=dev)
    phys = dinv.physics.Blur(filter=k3, padding="circular", device=dev)
    for bad in (torch.rand(2, 1, 8, device=dev), torch.rand(1, 1, 2, 2, 2, 2, device=dev)):
        for fn in (phys.A, phys.A_adjoint):
            with pytest.raises(ValueError, match="Expected Tensor dimension to be 4 or 5"):
                fn(bad)
    with pytest.raises(ValueError, match="Input and filter must be 5D tensors"):
        dinv.physics.Blur(filter=torch.rand(1, 1, 3, 3, device=dev), padding="circular", device=dev).A(x)
    with pytest.raises(AssertionError):
        dinv.physics.Blur(filter=torch.rand(3, 1, 3, 3, 3, device=dev), device=dev).A(x)
    with pytest.raises(AssertionError):
        dinv.physics.Blur(filter=torch.rand(1, 2, 3, 3, 3, device=dev), device=dev).A(x)
    # filter= is stored as the buffer; use_fft is stored and runs the same kernel
    k2 = torch.rand(1, 1, 3, 5, 3, device=dev)
    y = phys.A(x, filter=k2)
    assert phys.filter is not None and torch.equal(phys.filter, k2)
    f = dinv.physics.Blur(filter=k2, padding="circular", use_fft=True, device=dev)
    assert f.use_fft and torch.equal(f.A(x), y)
    # a 4-D input with a 4-D filter still takes the 2-D kernel
    n0 = dinv.launch_count()
    dinv.physics.Blur(filter=torch.rand(1, 1, 3, 3, device=dev), padding="circular", device=dev).A(torch.rand(1, 1, 8, 8, device=dev))
    assert dinv.launch_count() - n0 == 1


def test_autograd_through_opposite_kernel(dev):
    import deepinv_b200 as dinv

    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2, 5, 12, 10, generator=g).to(dev).requires_grad_()
    k = torch.randn(1, 2, 3, 4, 3, generator=g).to(dev)
    for pad in PADS:
        phys = dinv.physics.Blur(filter=k, padding=pad, device=dev)
        y = phys.A(x)
        r = torch.randn(y.shape, generator=g).to(dev)
        (gx,) = torch.autograd.grad((y * r).sum(), x)
        assert rel_err(gx, phys.A_adjoint(r)) < 1e-6, pad
        # and the adjoint's gradient is A
        v = torch.randn(y.shape, generator=g).to(dev).requires_grad_()
        s = torch.randn(x.shape, generator=g).to(dev)
        (gv,) = torch.autograd.grad((phys.A_adjoint(v) * s).sum(), v)
        assert rel_err(gv, phys.A(s)) < 1e-6, pad


def test_algorithms(dev):
    """CG prox_l2, PGD with Tikhonov and GD with ZeroPrior on a 3-D circular blur against the reference's runs, and the
    power-method norm against the fp64 one"""
    import deepinv_b200 as dinv
    from deepinv_b200.optim import GD, L2, PGD, Tikhonov, ZeroPrior

    g = load_golden("blur3d_algo")
    phys = dinv.physics.Blur(filter=g["k"].to(dev), padding="circular", device=dev)
    phys.max_iter, phys.tol = int(g["max_iter"]), float(g["tol"])
    y = g["y"].to(dev)
    with torch.no_grad():
        prox = phys.prox_l2(g["z"].to(dev), y, float(g["gamma"]))
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
        gd = GD(data_fidelity=L2(), prior=ZeroPrior(), stepsize=1.0, max_iter=6, early_stop=False)(y, phys)
        dag = phys.A_dagger(y)
        norm = float(phys.compute_norm(torch.rand(g["x"].shape, device=dev), max_iter=200, tol=1e-7, verbose=False))
    assert rel_err(prox, g["prox"]) < 1e-4
    assert rel_err(pgd, g["pgd"]) < TOL
    assert rel_err(gd, g["gd"]) < TOL
    assert rel_err(phys.A(dag), y) < 0.1  # a least-squares solution: the residual is the noise's share outside the range
    kf = torch.fft.fftn(g["k"][0, 0].double(), s=tuple(g["x"].shape[-3:]))  # circular: |A|^2 = max |k^|^2
    assert abs(norm - float(kf.abs().max() ** 2)) < 0.05 * norm
