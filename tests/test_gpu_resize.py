"""The MATLAB-bicubic resize on the H100: `DownsamplingMatlab`, `Upsampling` and `imresize_matlab` against the reference's golden
vectors, the fused kernels against the fp64 restatement (tests/resize_ref64.py) at user sizes, run-to-run bitwise results,
gradients, a PGD super-resolution run and argument errors."""
import pytest
import torch

import resize_ref64 as R
from conftest import golden_names, load_golden, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
ERRORS = (RuntimeError, ValueError, AssertionError, NotImplementedError, IndexError)


def cu(t):
    return t.to(DEV)


@pytest.mark.parametrize("name", golden_names("resize_f"))
def test_downsampling_matlab_golden(name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    f = float(g["factor"])
    p = dinv.physics.DownsamplingMatlab(factor=f if f % 1 else int(f), antialiasing=bool(int(g["aa"])), device=DEV)
    assert p.factor == int(g["stored_factor"])
    assert rel_err(p.A(cu(g["x"])), g["y"]) < 1e-5
    at = p.A_adjoint(cu(g["v"]))
    assert at.shape == g["At"].shape and rel_err(at, g["At"]) < 1e-5
    with torch.no_grad():
        assert rel_err(p.A_dagger(cu(g["y"])), g["dagger"]) < 1e-4
        if int(g["prox_err"]) >= 0:
            with pytest.raises(ERRORS[int(g["prox_err"])]):
                p.prox_l2(cu(g["x"]), cu(g["y"]), 0.5)
        else:
            assert rel_err(p.prox_l2(cu(g["x"]), cu(g["y"]), 0.5), g["prox"]) < 1e-4
        assert rel_err(p.prox_l2(cu(g["z"]), cu(g["y"]), 0.5), g["prox_even"]) < 1e-4


@pytest.mark.parametrize("name", golden_names("resize_tiny_"))
def test_tiny_images_raise(name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    with pytest.raises(ERRORS[int(g["err"])]):
        dinv.physics.DownsamplingMatlab(factor=int(g["factor"])).A(cu(g["x"]))


def test_imresize_matlab_golden():
    import deepinv_b200 as dinv

    F = dinv.physics.functional
    g = load_golden("resize_up2")
    x = cu(g["x"])
    assert rel_err(F.imresize_matlab(x, scale=2), g["up2"]) < 1e-5
    assert rel_err(F.imresize_matlab(x, scale=2, antialiasing=False), g["up2_noaa"]) < 1e-5
    assert rel_err(F.imresize_matlab(x, sizes=(25, 17)), g["up_sizes"]) < 1e-5
    assert rel_err(F.imresize_matlab(x, sizes=(6, 9)), g["down_sizes"]) < 1e-5
    assert rel_err(F.imresize_matlab(cu(g["x3"]), scale=2), g["up2_3d"]) < 1e-5


@pytest.mark.parametrize("name", [n for n in golden_names("resize_upsampling_") if n != "resize_upsampling_valid"])
def test_upsampling_golden(name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    u = dinv.physics.Upsampling(img_size=(3, 16, 16), filter=cu(g["filter"]), factor=2, padding=name.rsplit("_", 1)[1],
                                device=DEV)
    assert rel_err(u.A(cu(g["x"])), g["y"]) < 1e-5
    assert rel_err(u.A_adjoint(cu(g["v"])), g["At"]) < 1e-5
    with torch.no_grad():
        if int(g["prox_err"]) >= 0:
            with pytest.raises(ERRORS[int(g["prox_err"])]):
                u.prox_l2(cu(g["x"]), cu(g["v"]), 0.5)
        else:
            assert rel_err(u.prox_l2(cu(g["x"]), cu(g["v"]), 0.5), g["prox"]) < 1e-4


@pytest.mark.parametrize("shape,factor", [((64, 3, 256, 256), 2), ((64, 3, 256, 256), 3), ((64, 3, 256, 256), 4),
                                          ((4, 3, 1080, 1920), 2), ((4, 3, 1080, 1920), 3)])
def test_user_sizes_against_fp64(shape, factor):
    """the kernels within 2x of the dense fp32 operator's distance to the fp64 one (plus a floor for exact cases)"""
    from deepinv_b200.physics.imresize import resize, resize_adjoint, resize_plan

    B, C, H, W = shape
    x = torch.rand(shape, generator=torch.Generator().manual_seed(factor), device="cpu").to(DEV)
    _, th, tw = resize_plan(H, W, scale=1 / factor)
    MH, MW = (m.to(DEV) for m in R.operators(H, W, 1 / factor))
    MH32, MW32 = (m.to(DEV) for m in R.operators(H, W, 1 / factor, dtype=torch.float32))
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        y = resize(x, th, tw)
        y64 = R.apply(x, MH, MW)
        e32 = rel_err(R.apply(x, MH32, MW32), y64)
        assert rel_err(y, y64) <= 2 * e32 + 1e-7
        v = torch.randn(y.shape, device=DEV)
        xt = resize_adjoint(v, th, tw, H, W)
        x64 = R.apply_t(v, MH, MW)
        e32t = rel_err(R.apply_t(v, MH32, MW32), x64)
        assert rel_err(xt, x64) <= 2 * e32t + 1e-7
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    # run to run: bitwise
    assert torch.equal(resize(x, th, tw), y) and torch.equal(resize_adjoint(v, th, tw, H, W), xt)


def test_autograd_through_A_and_A_adjoint():
    import deepinv_b200 as dinv

    p = dinv.physics.DownsamplingMatlab(factor=4, device=DEV)
    x = torch.randn(3, 2, 96, 128, device=DEV, requires_grad=True)
    w = torch.randn(3, 2, 24, 32, device=DEV)
    (gx,) = torch.autograd.grad((p.A(x) * w).sum(), x)
    assert torch.equal(gx, p.A_adjoint(w))
    v = w.clone().requires_grad_()
    u = torch.randn(3, 2, 96, 128, device=DEV)
    (gv,) = torch.autograd.grad((p.A_adjoint(v) * u).sum(), v)
    assert torch.equal(gv, p.A(u))
    # an unfolded-style step: gradients reach a parameter through the data term
    step = torch.tensor(0.5, device=DEV, requires_grad=True)
    y = p.A(torch.rand(3, 2, 96, 128, device=DEV))
    z = torch.zeros(3, 2, 96, 128, device=DEV)
    out = z - step * p.A_adjoint(p.A(z) - y)
    (gs,) = torch.autograd.grad(out.square().sum(), step)
    assert torch.isfinite(gs) and float(gs) != 0.0


def test_pgd_super_resolution_golden():
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("resize_pgd")
    p = dinv.physics.DownsamplingMatlab(factor=2, device=DEV)
    algo = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=float(g["stepsize"]), lambda_reg=float(g["lambda_reg"]),
               max_iter=int(g["max_iter"]), early_stop=False)
    n0 = dinv.launch_count()
    with torch.no_grad():
        out = algo(cu(g["y"]), p)
    torch.cuda.synchronize()
    assert dinv.launch_count() > n0
    assert rel_err(out, g["pgd"]) < 1e-5


def test_argument_errors():
    import deepinv_b200 as dinv

    F = dinv.physics.functional
    x = torch.rand(1, 3, 16, 16, device=DEV)
    with pytest.raises(ValueError):
        F.imresize_matlab(x)
    with pytest.raises(ValueError):
        F.imresize_matlab(x, scale=0.5, sizes=(8, 8))
    with pytest.raises(ValueError):
        F.imresize_matlab(x, scale=0.5, padding_type="zeros")
    with pytest.raises(NotImplementedError):
        F.imresize_matlab(x, scale=0.5, kernel="gaussian")
    with pytest.raises(NotImplementedError):
        F.imresize_matlab(x.double(), scale=0.5)
    with pytest.raises(dinv.DinvkError):
        F.imresize_matlab(x.cpu(), scale=0.5)  # no CPU fall-back
    with pytest.raises(AssertionError):
        dinv.physics.Upsampling(img_size=(3, 16, 16), padding="valid")
    p = dinv.physics.DownsamplingMatlab(factor=2, device=DEV)
    with pytest.raises(ValueError):
        p.A(torch.rand(1, 1, 3, 16, 16, device=DEV))
    # an empty batch launches nothing
    n0 = dinv.launch_count()
    assert p.A(torch.rand(0, 3, 16, 16, device=DEV)).shape == (0, 3, 8, 8)
    assert p.A_adjoint(torch.rand(0, 3, 8, 8, device=DEV)).shape == (0, 3, 16, 16)
    assert dinv.launch_count() == n0
