"""GPU: the tiled space-varying blur (libdinvk tiled_svblur_fwd_kernel / tiled_svblur_adj_kernel) through the package API,
against the reference's golden vectors (tests/golden/tiledsv_*.npz), an fp64 evaluation of the reference's per-patch
algorithm on the device (tests/tiledsv_oracle.py), and the existing Blur kernels.  Tolerance: 1e-5 relative L2 in fp32."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tiledsv_oracle as O  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402
from oracle import ref_ops as R  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-5
OPERATOR_CASES = [n for n in golden_names("tiledsv_") if n != "tiledsv_algo"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def geometry(g):
    return tuple(int(v) for v in g["patch"]), tuple(int(v) for v in g["stride"])


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name, dev):
    import deepinv_b200 as dinv

    g = load_golden(name)
    patch, stride = geometry(g)
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=g["h"].to(dev), patch_size=patch, stride=stride,
                                              blending_mode=O.MODES[int(g["mode"])], device=dev)
    assert rel_err(phys.A(g["x"].to(dev)), g["y"]) < TOL
    assert phys.multipliers.is_cuda and torch.equal(phys.multipliers.cpu(), g["w"])
    assert rel_err(phys.A_adjoint(g["v"].to(dev)), g["At"]) < TOL


def test_1024_per_sample_motion_psfs(dev):
    """(32, 1, 1024, 1024), patch 128, stride 64, K = 225 per-sample 31 x 31 motion PSFs; samples 0 and 1 against the
    reference's per-patch algorithm in fp64 on the device"""
    import deepinv_b200 as dinv
    from deepinv_b200.physics.generator import MotionBlurGenerator, TiledBlurGenerator

    gen = TiledBlurGenerator(MotionBlurGenerator((31, 31), device=dev), patch_size=128, stride=64, device=dev)
    h = gen.step(batch_size=32, img_size=(1024, 1024), seed=0)["filters"]
    assert h.shape == (32, 1, 225, 31, 31)
    x = torch.rand(32, 1, 1024, 1024, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=h, patch_size=128, stride=64, device=dev)
    with torch.no_grad():
        y = phys.A(x)
        v = torch.randn(y.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
        at = phys.A_adjoint(v)
    w = phys.multipliers.double()
    ref = O.tiledsv_A_patches(x[:2].double(), w, h[:2].double(), (128, 128), (64, 64))
    assert rel_err(y[:2], ref) < TOL
    x2 = x[:2].double().requires_grad_()
    (ref_at,) = torch.autograd.grad((O.tiledsv_A_patches(x2, w, h[:2].double(), (128, 128), (64, 64)) * v[:2].double()).sum(), x2)
    assert rel_err(at[:2], ref_at) < TOL
    lhs, rhs = float((y.double() * v.double()).sum()), float((x.double() * at.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs)


def test_small_k_against_blur_kernels(dev):
    """sum_k Wt_k . Blur_k.A(x) with the existing Blur kernels, K = 6 across several 64-pixel tiles"""
    import deepinv_b200 as dinv

    gen = torch.Generator(device=dev).manual_seed(3)
    H, W, patch, stride = 200, 150, (120, 90), (40, 60)
    nr, nc = O.num_patches(H, W, patch, stride)
    x = torch.randn(3, 2, H, W, device=dev, generator=gen)
    h = torch.rand(3, 1, nr * nc, 11, 9, device=dev, generator=gen)
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=h, patch_size=patch, stride=stride, device=dev)
    with torch.no_grad():
        y = phys.A(x)
        Wt = O.placed(phys.multipliers.cpu(), H, W, 11, 9, patch, stride).to(dev)
        ref = sum(Wt[k] * dinv.physics.Blur(filter=h[:, :, k].contiguous(), padding="valid", device=dev).A(x) for k in range(nr * nc))
    assert nr * nc == 6 and rel_err(y, ref) < TOL


def test_batch_independence_repeatability_graph_and_empty(dev):
    import deepinv_b200 as dinv

    gen = torch.Generator(device=dev).manual_seed(4)
    H, W, patch, stride = 260, 190, 64, 32
    nr, nc = O.num_patches(H, W, (patch, patch), (stride, stride))
    x = torch.randn(4, 1, H, W, device=dev, generator=gen)
    h = torch.rand(4, 1, nr * nc, 15, 15, device=dev, generator=gen)
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=h, patch_size=patch, stride=stride, device=dev)
    with torch.no_grad():
        y = phys.A(x)
        at = phys.A_adjoint(y)
        assert torch.equal(phys.A(x), y) and torch.equal(phys.A_adjoint(y), at)
        for b in range(4):
            assert torch.equal(phys.A(x[b: b + 1], filters=h[b: b + 1]), y[b: b + 1])
            assert torch.equal(phys.A_adjoint(y[b: b + 1]), at[b: b + 1])
        phys.update_parameters(filters=h)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            phys.A_adjoint(phys.A(x))
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = phys.A_adjoint(phys.A(x))
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, at)
    phys.update_parameters(filters=h[:1])  # filters shared over the batch: an empty batch broadcasts
    n0 = dinv.launch_count()
    empty = phys.A(torch.empty(0, 1, H, W, device=dev))
    assert empty.shape == (0, 1, H - 14, W - 14) and dinv.launch_count() == n0
    assert phys.A_adjoint(torch.empty(0, 1, H - 14, W - 14, device=dev)).shape == (0, 1, H, W) and dinv.launch_count() == n0


def test_pgd_and_cg_prox_against_oracle(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("tiledsv_algo")
    patch, stride = geometry(g)
    H, W = g["x"].shape[-2:]
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=g["h"].to(dev), patch_size=patch, stride=stride, device=dev)
    y = g["y"].to(dev)
    with torch.no_grad():
        prox = phys.prox_l2(g["z"].to(dev), y, float(g["gamma"]))
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
    assert rel_err(prox, g["prox"]) < TOL and rel_err(pgd, g["pgd"]) < TOL
    w = phys.multipliers.cpu()
    A = lambda v: O.tiledsv_A(v, w, g["h"], patch, stride)
    At = lambda v: O.tiledsv_At(v, w, g["h"], patch, stride, H, W)
    xp, _ = R.prox_l2_cg(A, At, g["z"], g["y"], float(g["gamma"]), max_iter=int(g["max_iter"]), tol=float(g["tol"]))
    assert rel_err(prox, xp) < TOL
    assert rel_err(pgd, R.pgd(g["y"], A, At, lambda v, s: v / 1.1, 1.0, None, 6)) < TOL
