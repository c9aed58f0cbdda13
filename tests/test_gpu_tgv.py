"""GPU: the TGV prox and stencils (libdinvk tv.cu) through the package API, against the reference's golden vectors
(tests/golden/tgv_*.npz) and the torch oracle (tests/tgv_oracle.py) evaluated on the CPU.  Tolerance: 1e-5 relative L2
in fp32; where that is not met, the kernel must be no farther from an fp64 oracle run than the fp32 oracle is."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tgv_oracle as O  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
DENOISER_CASES = [n for n in golden_names("tgv_") if n not in ("tgv_stencils", "tgv_algo_blur")]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _ths(z, dev):
    return z["ths"].to(dev) if z["ths"].dim() else float(z["ths"])


def _close(a, b, fp64=None):
    """a within TOL of the golden b, or (for a state field that needs more) no farther from the fp64 oracle than b is"""
    a = a.cpu()
    if torch.isnan(b).all():
        return torch.isnan(a).all()
    if rel_err(a, b) < TOL:
        return True
    ref = fp64()
    return rel_err(a, ref) <= rel_err(b, ref)


@pytest.mark.parametrize("name", DENOISER_CASES)
def test_golden_denoiser_with_warm_restart(name, dev):
    import deepinv_b200 as dinv

    z = load_golden(name)
    den = dinv.models.TGVDenoiser(n_it_max=int(z["n_it_max"]), crit=float(z["crit"]))
    # torch's CPU sqrt is not always correctly rounded and the kernel's is, so the dual state u2 (1e-7 level differences
    # amplified over hundreds of iterations) is allowed the fp64 yardstick; the fp64 oracle runs the golden counts
    ths64 = z["ths"].double() if z["ths"].dim() else float(z["ths"])
    memo = {}

    def fp64():
        if not memo:
            s1 = O.tgv_denoise(z["y"].double(), ths64, n_it_max=int(z["n_iter1"]), crit=0.0)
            s2 = O.tgv_denoise(z["y2"].double(), ths64, n_it_max=int(z["n_iter2"]), crit=0.0, x2=s1[0], r2=s1[1], u2=s1[2])
            memo.update(s1=s1, s2=s2)
        return memo

    out1 = den(z["y"].to(dev), _ths(z, dev))
    assert int(den.n_iter) == int(z["n_iter1"]) and den.has_converged == bool(z["converged1"])
    assert den.x2.shape == z["y"].shape and den.r2.shape == (*z["y"].shape, 2) and den.u2.shape == (*z["y"].shape, 4)
    assert not den.u2.requires_grad
    assert _close(out1, z["out1"]) and _close(den.r2, z["r2_1"])
    assert _close(den.u2, z["u2_1"], lambda: fp64()["s1"][2])
    out2 = den(z["y2"].to(dev), _ths(z, dev))  # warm restart from the first call's state
    assert int(den.n_iter) == int(z["n_iter2"]) and den.has_converged == bool(z["converged2"])
    assert _close(out2, z["out2"]) and _close(den.r2, z["r2_2"])
    assert _close(den.u2, z["u2_2"], lambda: fp64()["s2"][2])


def test_golden_stencils(dev):
    import deepinv_b200 as dinv

    z = load_golden("tgv_stencils")
    D = dinv.models.TGVDenoiser
    assert torch.equal(D.epsilon(z["f"].to(dev)).cpu(), z["epsilon"])
    assert torch.equal(D.epsilon_adjoint(z["gfield"].to(dev)).cpu(), z["epsilon_adjoint"])
    x = torch.randn(2, 3, 14, 19, device=dev)
    assert torch.equal(D.nabla(x).cpu(), O.tv_nabla(x.cpu()))
    with pytest.raises(ValueError):
        D.epsilon(x)
    with pytest.raises(ValueError):
        D.epsilon_adjoint(x)


def test_golden_pnp_pgd_on_circular_blur(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP

    z = load_golden("tgv_algo_blur")
    phys = dinv.physics.Blur(filter=z["filt"].to(dev), padding="circular", device=dev)
    with torch.no_grad():
        pgd = PGD(data_fidelity=L2(), prior=PnP(dinv.models.TGVDenoiser(n_it_max=100, crit=1e-5)), stepsize=1.0,
                  sigma_denoiser=0.05, max_iter=5, early_stop=False)(z["y"].to(dev), phys)
    assert rel_err(pgd, z["pgd"]) < TOL


def _image(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.linspace(0, 1, W).expand(H, W) + torch.linspace(0, 0.5, H)[:, None]
    return (base + 0.3 * torch.randn(B, C, H, W, generator=g)).float()


@pytest.mark.parametrize("shape,ths,crit,n_it_max", [
    ((4, 3, 300, 257), "per-sample", 0.0, 30),
    ((2, 1, 1024, 1024), 0.1, 0.0, 20),
    ((64, 2, 256, 256), 0.1, 1e-5, 20),  # the cfg2 shape
])
def test_large_against_cpu_oracle(shape, ths, crit, n_it_max, dev):
    import deepinv_b200 as dinv

    y = _image(*shape, seed=shape[0])
    lam = torch.linspace(0.05, 0.3, shape[0]) if ths == "per-sample" else ths
    den = dinv.models.TGVDenoiser(n_it_max=n_it_max, crit=crit)
    out = den(y.to(dev), lam.to(dev) if isinstance(lam, torch.Tensor) else lam).cpu()
    n = int(den.n_iter)
    xr, _, _, nr, _ = O.tgv_denoise(y, lam, n_it_max=n_it_max, crit=crit)
    assert n == nr
    e = rel_err(out, xr)
    if e >= TOL:
        x64, _, _, _, _ = O.tgv_denoise(y.double(), lam.double() if isinstance(lam, torch.Tensor) else lam, n_it_max=n, crit=0.0)
        assert rel_err(out, x64) <= rel_err(xr, x64), (e, rel_err(out, x64), rel_err(xr, x64))


def _state(y):
    return y, torch.zeros(*y.shape, 2, device=y.device), torch.zeros(*y.shape, 4, device=y.device)


def _consts(lam):
    return 0.01 * (lam * 0.1), lam * 0.15


def test_replay_is_the_run_stopped_at_the_break(dev):
    from deepinv_b200 import ops

    y = _image(4, 1, 200, 150, seed=12)
    x0 = torch.zeros_like(y)  # from x2 = 0 without over-relaxation rel_err falls steadily
    rels = []
    O.tgv_denoise(y, 0.15, rho=1.0, x2=x0, n_it_max=64, crit=0.0, rels=rels)
    yd = y.to(dev)
    tl1, l2 = _consts(torch.full((4,), 0.15, device=dev))
    _, r0, u0 = _state(yd)
    _, K = ops.tgv_block()
    for mod in sorted({0, K - 2, K - 1}):
        i = next(i for i in range(max(K, 3), 64) if i % K == mod and rels[i] < 0.99 * min(rels[2:i]))
        crit = (rels[i] * min(rels[2:i])) ** 0.5
        stats = {}
        x, r, u, n = ops.tgv_prox(yd, tl1, l2, x0.to(dev), r0, u0, rho=1.0, n_it_max=64, crit=crit, stats=stats)
        assert int(n) == i + 1 and stats["converged"]
        xs, rs, us, _ = ops.tgv_prox(yd, tl1, l2, x0.to(dev), r0, u0, rho=1.0, n_it_max=i + 1, crit=0.0)
        assert torch.equal(x, xs) and torch.equal(r, rs) and torch.equal(u, us)


def test_batch_independence_bitwise(dev):
    from deepinv_b200 import ops

    y = _image(5, 2, 130, 97, seed=14).to(dev)
    lam = torch.linspace(0.05, 0.4, 5, device=dev)
    tl1, l2 = _consts(lam)
    x, r, u, _ = ops.tgv_prox(y, tl1, l2, *_state(y), n_it_max=25, crit=0.0)
    for b in range(5):
        yb = y[b:b + 1]
        xb, rb, ub, _ = ops.tgv_prox(yb, tl1[b:b + 1], l2[b:b + 1], *_state(yb), n_it_max=25, crit=0.0)
        assert torch.equal(xb, x[b:b + 1]) and torch.equal(rb, r[b:b + 1]) and torch.equal(ub, u[b:b + 1])


def test_reference_convergence_case(dev):
    """the reference's own TGV convergence check: n_it_max = 5000, crit = 1e-4, ths = 2.0 converges"""
    import deepinv_b200 as dinv

    y = _image(1, 1, 64, 64, seed=15)
    den = dinv.models.TGVDenoiser(n_it_max=5000, crit=1e-4)
    out = den(y.to(dev), ths=2.0)
    n = int(den.n_iter)
    assert den.has_converged and n < 5000
    xr, _, _, nr, rel_at_break = O.tgv_denoise(y, 2.0, n_it_max=5000, crit=1e-4)
    if abs(rel_at_break - 1e-4) > 0.01 * 1e-4:
        assert n == nr, (n, nr, rel_at_break)
    if n != nr:  # the break test sits on the edge (here within 0.3 % of crit): compare at the kernel's iteration count
        xr, _, _, _, _ = O.tgv_denoise(y, 2.0, n_it_max=n, crit=0.0)
    assert rel_err(out, xr) < TOL


def test_errors_and_empty(dev):
    import deepinv_b200 as dinv
    from deepinv_b200 import ops

    den = dinv.models.TGVDenoiser()
    with pytest.raises(RuntimeError):
        den(torch.zeros(1, 1, 8, 8, device=dev))
    with pytest.raises(NotImplementedError):
        den(torch.zeros(1, 1, 4, 8, 8, device=dev), 0.1)
    with pytest.raises(NotImplementedError):
        den(torch.zeros(1, 1, 8, 8, device=dev, requires_grad=True), 0.1)
    out = dinv.models.TGVDenoiser(n_it_max=0, ths=0.1)(torch.ones(1, 1, 8, 8, device=dev))
    assert torch.equal(out, torch.ones(1, 1, 8, 8, device=dev))
    y = torch.zeros(0, 1, 8, 8, device=dev)
    stats = {}
    x, r, u, n = ops.tgv_prox(y, torch.zeros(0, device=dev), torch.zeros(0, device=dev), *_state(y), stats=stats)
    assert x.shape == y.shape and r.shape == (0, 1, 8, 8, 2) and u.shape == (0, 1, 8, 8, 4)
    assert int(n) == 0 and stats["launches"] == 0
