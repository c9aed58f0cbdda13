"""GPU: the space-varying blur (libdinvk svblur_fwd_kernel / svblur_adj_kernel) through the package API, against the
reference's golden vectors (tests/golden/svblur_*.npz), the oracle (tests/svblur_oracle.py) on the CPU, and the existing
Blur kernels.  Tolerance: 1e-5 relative L2 in fp32."""
import sys
import warnings
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import svblur_oracle as O  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402
from oracle import ref_ops as R  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
OPERATOR_CASES = [n for n in golden_names("svblur_") if n != "svblur_algo"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _phys(g, dev):
    import deepinv_b200 as dinv

    return dinv.physics.SpaceVaryingBlur(filters=g["h"], multipliers=g["w"], padding=O.PADS[int(g["pad"])],
                                         use_fft=bool(g["use_fft"]) if "use_fft" in g else False, device=dev)


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name, dev):
    g = load_golden(name)
    phys = _phys(g, dev)
    assert rel_err(phys.A(g["x"].to(dev)), g["y"]) < TOL
    assert rel_err(phys.A_adjoint(g["v"].to(dev)), g["At"]) < TOL


def _large_case(dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(32, 1, 1024, 1024, device=dev, generator=gen)
    w = torch.rand(1, 1, 10, 1024, 1024, device=dev, generator=gen)
    h = torch.rand(1, 1, 10, 31, 31, device=dev, generator=gen)
    return x, w / w.sum(2, keepdim=True), h / h.sum((-2, -1), keepdim=True)


def _oracle_A(x, w, h, pad):
    """the CPU oracle; circular as the valid oracle blur of the circularly padded product (the reference's own F.pad route),
    which keeps one 1024 x 1024 image with K = 10 at 31 x 31 taps within seconds"""
    if pad == "valid":
        return O.svblur_A(x, w, h, "valid")
    fh, fw = h.shape[-2:]
    out = 0.0
    for k in range(w.size(2)):
        p = torch.nn.functional.pad(w[:, :, k] * x, (fw - 1 - fw // 2, fw // 2, fh - 1 - fh // 2, fh // 2), mode="circular")
        out = out + R.blur_A(p, h[:, :, k], "valid")
    return out


@pytest.mark.parametrize("pad", ["circular", "valid"])
def test_large_against_blur_sum_and_oracle(pad, dev):
    import deepinv_b200 as dinv
    from deepinv_b200 import _ffi, ops

    x, w, h = _large_case(dev, 0)
    phys = dinv.physics.SpaceVaryingBlur(filters=h, multipliers=w, padding=pad, device=dev)
    with torch.no_grad():
        y = phys.A(x)
        code = _ffi.PADDING_CODES[pad]
        ref = sum(ops.blur_fwd(w[:, :, k] * x, h[:, :, k], code) for k in range(10))
    assert rel_err(y, ref) <= 2e-6  # only the order of the k sum differs
    i = 0 if pad == "circular" else 31
    assert rel_err(y[i:i + 1], _oracle_A(x[i:i + 1].cpu(), w.cpu(), h.cpu(), pad)) < TOL


@pytest.mark.parametrize("pad", ["valid", "circular", "replicate", "reflect", "constant"])
def test_adjointness(pad, dev):
    import deepinv_b200 as dinv

    gen = torch.Generator(device=dev).manual_seed(5)
    B, C, H, W, K = 2, 3, 70, 131, 4
    x = torch.randn(B, C, H, W, device=dev, generator=gen)
    w = torch.rand(B, 1, K, H, W, device=dev, generator=gen)
    h = torch.rand(1, C, K, 7, 6, device=dev, generator=gen)
    phys = dinv.physics.SpaceVaryingBlur(filters=h, multipliers=w, padding=pad, device=dev)
    y = phys.A(x)
    v = torch.randn(y.shape, device=dev, generator=gen)
    lhs, rhs = float((y.double() * v.double()).sum()), float((x.double() * phys.A_adjoint(v).double()).sum())
    assert abs(lhs - rhs) <= TOL * abs(lhs)


@pytest.mark.parametrize("pad", ["circular", "reflect"])
def test_bitwise_batch_independent_and_repeatable(pad, dev):
    from deepinv_b200 import _ffi, ops

    gen = torch.Generator(device=dev).manual_seed(6)
    B, C, H, W, K = 3, 2, 96, 80, 3
    x = torch.randn(B, C, H, W, device=dev, generator=gen)
    w = torch.rand(B, C, K, H, W, device=dev, generator=gen)
    h = torch.rand(1, 1, K, 9, 8, device=dev, generator=gen)
    code = _ffi.PADDING_CODES[pad]
    y = ops.svblur_fwd(x, w, h, code)
    at = ops.svblur_adj(y, w, h, code, H, W)
    assert torch.equal(y, ops.svblur_fwd(x, w, h, code)) and torch.equal(at, ops.svblur_adj(y, w, h, code, H, W))
    for b in range(B):
        assert torch.equal(ops.svblur_fwd(x[b:b + 1], w[b:b + 1], h, code), y[b:b + 1])
        assert torch.equal(ops.svblur_adj(y[b:b + 1], w[b:b + 1], h, code, H, W), at[b:b + 1])


@pytest.mark.parametrize("fsize", [31, 90])
def test_one_term_unit_multiplier_is_blur(fsize, dev):
    """K = 1, w = 1 is Blur bitwise; 90 x 90 taps take the forward path that re-reads x for every term"""
    from deepinv_b200 import _ffi, ops

    gen = torch.Generator(device=dev).manual_seed(fsize)
    x = torch.randn(2, 1, 200, 264, device=dev, generator=gen)
    h = torch.rand(1, 1, 1, fsize, fsize, device=dev, generator=gen)
    w = torch.ones(1, 1, 1, 200, 264, device=dev)
    for pad in ("circular", "valid", "reflect"):
        code = _ffi.PADDING_CODES[pad]
        y = ops.svblur_fwd(x, w, h, code)
        assert torch.equal(y, ops.blur_fwd(x, h[:, :, 0], code)), pad
        assert torch.equal(ops.svblur_adj(y, w, h, code, 200, 264), ops.blur_adj(y, h[:, :, 0], code, 200, 264)), pad


def test_cuda_graph_replay_and_empty_batch(dev):
    import deepinv_b200 as dinv

    gen = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(2, 1, 130, 100, device=dev, generator=gen)
    w = torch.rand(1, 1, 4, 130, 100, device=dev, generator=gen)
    h = torch.rand(1, 1, 4, 11, 11, device=dev, generator=gen)
    phys = dinv.physics.SpaceVaryingBlur(filters=h, multipliers=w, padding="reflect", device=dev)
    with torch.no_grad():
        eager = phys.A_adjoint(phys.A(x))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            phys.A_adjoint(phys.A(x))  # warm-up: workspace allocation outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = phys.A_adjoint(phys.A(x))
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)
    n0 = dinv.launch_count()
    empty = phys.A(torch.empty(0, 1, 130, 100, device=dev))
    assert empty.shape == (0, 1, 130, 100) and dinv.launch_count() == n0
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        phys.update_parameters(filters=h.cpu())
    assert any("different device" in str(c.message) for c in caught) and phys.filters.is_cuda


def test_pgd_and_admm_against_oracle(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import ADMM, L2, PGD, Tikhonov

    g = load_golden("svblur_algo")
    pad = O.PADS[int(g["pad"])]
    H, W = g["x"].shape[-2:]
    phys = dinv.physics.SpaceVaryingBlur(filters=g["h"], multipliers=g["w"], padding=pad, device=dev)
    y = g["y"].to(dev)
    with torch.no_grad():
        assert rel_err(phys.prox_l2(g["z"].to(dev), y, float(g["gamma"])), g["prox"]) < TOL
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
        admm = ADMM(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=3, early_stop=False)(y, phys)
    assert rel_err(pgd, g["pgd"]) < TOL
    A = lambda v: O.svblur_A(v, g["w"], g["h"], pad)
    At = lambda v: O.svblur_At(v, g["w"], g["h"], pad, H, W)
    prox = lambda v, gam: R.prox_l2_cg(A, At, v, g["y"], gam, max_iter=int(g["max_iter"]), tol=float(g["tol"]))[0]
    assert rel_err(admm, R.admm(g["y"], prox, At, lambda v, s: v / 1.1, 1.0, None, 3)) < 1e-4
