"""GPU: the TV prox, stencils and priors (libdinvk tv.cu) through the package API, against the reference's golden vectors
(tests/golden/tv_*.npz) and the torch oracle (tests/tv_oracle.py) evaluated on the CPU.  Tolerance: 1e-5 relative L2 in
fp32; where that is not met, the kernel must be no farther from an fp64 oracle run than the fp32 oracle is."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tv_oracle as O  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
DENOISER_CASES = [n for n in golden_names("tv_") if n.startswith(("tv_iso", "tv_l1"))]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _ths(z, dev):
    return z["ths"].to(dev) if z["ths"].dim() else float(z["ths"])


@pytest.mark.parametrize("name", DENOISER_CASES)
def test_golden_denoiser_with_warm_restart(name, dev):
    import deepinv_b200 as dinv

    z = load_golden(name)
    cls = dinv.models.TVL1Denoiser if int(z["l1"]) else dinv.models.TVDenoiser
    den = cls(n_it_max=int(z["n_it_max"]), crit=float(z["crit"]))
    out1 = den(z["y"].to(dev), _ths(z, dev))
    assert int(den.n_iter) == int(z["n_iter1"])
    assert rel_err(out1, z["out1"]) < TOL
    assert den.x2.shape == z["y"].shape and den.u2.shape == (*z["y"].shape, 2) and not den.u2.requires_grad
    u_ref = z["u2_1"]
    read = torch.zeros_like(u_ref, dtype=torch.bool)  # the components nabla_adjoint reads (the rest is NaN when ths = 0)
    read[:, :, :-1, :, 0] = True
    read[:, :, :, :-1, 1] = True
    assert rel_err(den.u2.cpu()[read], u_ref[read]) < TOL
    out2 = den(z["y2"].to(dev), _ths(z, dev))  # warm restart from the first call's state
    assert int(den.n_iter) == int(z["n_iter2"])
    assert rel_err(out2, z["out2"]) < TOL


def test_golden_prior_functions(dev):
    import deepinv_b200 as dinv

    z = load_golden("tv_prior")
    x, gf = z["x"].to(dev), z["gfield"].to(dev)
    p, p1 = dinv.optim.TVPrior(), dinv.optim.TVL1Prior()
    assert torch.equal(p.nabla(x).cpu(), z["nabla"])
    assert torch.equal(p.nabla_adjoint(gf).cpu(), z["nabla_adjoint"])
    assert rel_err(p.grad(x), z["grad"]) < TOL
    assert rel_err(p.fn(x), z["fn"]) < TOL
    assert rel_err(p1.fn(x), z["fn_l1"]) < TOL
    assert torch.equal(dinv.models.TVDenoiser.nabla(x).cpu(), z["nabla"])


def test_golden_pgd_and_pdcp_on_circular_blur(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PDCP, PGD, TVPrior

    z = load_golden("tv_algo_blur")
    phys = dinv.physics.Blur(filter=z["filt"].to(dev), padding="circular", device=dev)
    y = z["y"].to(dev)
    with torch.no_grad():
        pgd = PGD(data_fidelity=L2(), prior=TVPrior(n_it_max=200), stepsize=1.0, lambda_reg=0.05, max_iter=5, early_stop=False)(y, phys)
        pdcp = PDCP(data_fidelity=L2(), prior=TVPrior(n_it_max=200), lambda_reg=0.05, stepsize=0.5, stepsize_dual=0.5, max_iter=5,
                    early_stop=False)(y, phys)
    assert rel_err(pgd, z["pgd"]) < TOL
    assert rel_err(pdcp, z["pdcp"]) < TOL


def _image(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.linspace(0, 1, W).expand(H, W) + torch.linspace(0, 0.5, H)[:, None]
    return (base + 0.3 * torch.randn(B, C, H, W, generator=g)).float()


@pytest.mark.parametrize("shape,ths,crit,n_it_max,l1", [
    ((64, 2, 256, 256), 0.1, 1e-5, 60, False),   # the cfg2 shape
    ((64, 2, 256, 256), 0.1, 2e-3, 60, True),
    ((4, 1, 1024, 1024), "per-sample", 1e-5, 40, False),
])
def test_large_against_cpu_oracle(shape, ths, crit, n_it_max, l1, dev):
    import deepinv_b200 as dinv

    y = _image(*shape, seed=shape[0])
    lam = torch.linspace(0.05, 0.3, shape[0]) if ths == "per-sample" else ths
    den = (dinv.models.TVL1Denoiser if l1 else dinv.models.TVDenoiser)(n_it_max=n_it_max, crit=crit)
    out = den(y.to(dev), lam.to(dev) if isinstance(lam, torch.Tensor) else lam).cpu()
    n = int(den.n_iter)
    xr, _, nr, rel_at_break = O.tv_denoise(y, lam, l1=l1, n_it_max=n_it_max, crit=crit)
    if abs(rel_at_break - crit) > 0.01 * crit:
        assert n == nr, (n, nr, rel_at_break)
    if n != nr:  # the break test sits on the edge: compare at the kernel's iteration count
        xr, _, _, _ = O.tv_denoise(y, lam, l1=l1, n_it_max=n, crit=0.0)
    e = rel_err(out, xr)
    if e >= TOL:
        x64, _, _, _ = O.tv_denoise(y.double(), lam.double() if isinstance(lam, torch.Tensor) else lam, l1=l1, n_it_max=n, crit=0.0)
        assert rel_err(out, x64) <= rel_err(xr, x64), (e, rel_err(out, x64), rel_err(xr, x64))


def test_run_to_run_bitwise(dev):
    import deepinv_b200 as dinv
    from deepinv_b200 import ops

    y = _image(8, 2, 300, 270, seed=11).to(dev)
    lam = torch.linspace(0.05, 0.2, 8, device=dev)
    u0 = torch.zeros(*y.shape, 2, device=dev)
    runs = [ops.tv_prox(y, lam, y, u0, n_it_max=100, crit=1e-4) for _ in range(3)]
    for x, u, n in runs[1:]:
        assert torch.equal(x, runs[0][0]) and torch.equal(u, runs[0][1]) and int(n) == int(runs[0][2])
    den = dinv.models.TVDenoiser(n_it_max=50, crit=0.0)
    assert torch.equal(den(y, 0.1), dinv.models.TVDenoiser(n_it_max=50, crit=0.0)(y, 0.1))


def test_replay_is_the_run_stopped_at_the_break(dev):
    from deepinv_b200 import ops

    y = _image(4, 1, 200, 150, seed=12).to(dev)
    lam = torch.full((4,), 0.15, device=dev)
    u0 = torch.zeros(*y.shape, 2, device=dev)
    rels = []
    O.tv_denoise(y.cpu(), 0.15, rho=1.0, n_it_max=64, crit=0.0, rels=rels)
    _, K = ops.tv_block()
    for mod in (0, K - 2, K - 1):
        i = next(i for i in range(K, 64) if i % K == mod and rels[i] < 0.995 * min(rels[2:i]))
        crit = (rels[i] * min(rels[2:i])) ** 0.5
        stats = {}
        x, u, n = ops.tv_prox(y, lam, y, u0, rho=1.0, n_it_max=64, crit=crit, stats=stats)
        assert int(n) == i + 1
        x0, u0_, _ = ops.tv_prox(y, lam, y, u0, rho=1.0, n_it_max=i + 1, crit=0.0)
        assert torch.equal(x, x0) and torch.equal(u, u0_)


def test_pgd_tv_prior_on_mri_against_oracle(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, TVPrior
    from oracle import ref_ops as R

    B, H, W = 2, 64, 48
    g = torch.Generator().manual_seed(3)
    x = _image(B, 2, H, W, seed=13)
    mask = (torch.rand(B, 1, 1, W, generator=g) > 0.5).float().expand(B, 2, H, W).contiguous()
    y = R.mri_A(x, mask)
    state = {}

    def tv_prox(v, _sigma):  # TVPrior.prox with its warm restart: gamma = lambda_reg * stepsize
        state["x2"], state["u2"], _, _ = O.tv_denoise(v, 0.05, n_it_max=300, crit=1e-8, x2=state.get("x2"), u2=state.get("u2"))
        return state["x2"]

    ref = R.pgd(y, lambda v: R.mri_A(v, mask), lambda v: R.mri_At(v, mask), tv_prox, 1.0, None, 4)
    phys = dinv.physics.MRI(mask=mask.to(dev), img_size=(2, H, W), device=dev)
    with torch.no_grad():
        out = PGD(data_fidelity=L2(), prior=TVPrior(n_it_max=300), stepsize=1.0, lambda_reg=0.05, max_iter=4, early_stop=False)(
            y.to(dev), phys)
    assert rel_err(out, ref) < TOL


def test_errors(dev):
    import deepinv_b200 as dinv

    den = dinv.models.TVDenoiser()
    with pytest.raises(RuntimeError):
        den(torch.zeros(1, 1, 8, 8, device=dev))
    with pytest.raises(NotImplementedError):
        den(torch.zeros(1, 1, 4, 8, 8, device=dev), 0.1)
    with pytest.raises(NotImplementedError):
        den(torch.zeros(1, 1, 8, 8, device=dev, requires_grad=True), 0.1)
    out = dinv.models.TVDenoiser(n_it_max=0, ths=0.1)(torch.ones(1, 1, 8, 8, device=dev))
    assert torch.equal(out, torch.ones(1, 1, 8, 8, device=dev))
