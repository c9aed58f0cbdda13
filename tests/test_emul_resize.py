"""The MATLAB-bicubic resize kernels (resize_fwd_kernel / resize_adj_kernel in deepinv_b200/csrc/blur.cu) on the host emulation.

Checked against the fp64 restatement (tests/resize_ref64.py) on every factor / antialiasing / odd-size case, on tiles that
cross every border, for adjointness in fp64, on an empty batch and on bad arguments; and through the package's own
`DownsamplingMatlab`, `Upsampling` and `imresize_matlab` against the reference's golden vectors (tests/golden/resize_*.npz),
with the emulated library behind `ops`.
"""
import ctypes
import math

import pytest
import torch

import resize_ref64 as R
from conftest import golden_names, load_golden, rel_err
from emul_util import emul_lib, ptr

EINVAL, EUNSUPPORTED = 1, 4
ERRORS = (RuntimeError, ValueError, AssertionError, NotImplementedError, IndexError)


@pytest.fixture
def emul_ops(monkeypatch):
    from deepinv_b200 import ops

    lib = emul_lib()

    def check(rc):
        assert rc == 0, lib.dinvk_last_error()

    monkeypatch.setattr(ops, "_require_cuda", lambda *ts: torch.device("cpu"))
    monkeypatch.setattr(ops, "_stream", lambda dev: None)
    monkeypatch.setattr(ops, "get_lib", lambda: lib)
    monkeypatch.setattr(ops, "check", check)
    ops._ws_cache.clear()
    yield lib
    ops._ws_cache.clear()


def table_matrix(n, m, scale, aa):
    from deepinv_b200.physics.imresize import axis_table

    t = axis_table(n, m, scale, aa)
    j = t.base.long()[:, None] + torch.arange(t.k)[None, :]
    j = torch.where(j < 0, -1 - j, torch.where(j >= n, 2 * n - 1 - j, j))
    return torch.zeros(m, n, dtype=torch.float64).scatter_add_(1, j, t.weight.double())


def run(x, scale, aa=True):
    from deepinv_b200.physics.imresize import resize, resize_adjoint, resize_plan

    H, W = x.shape[-2:]
    _, th, tw = resize_plan(H, W, scale=scale, antialiasing=aa)
    y = resize(x, th, tw)
    v = torch.randn(y.shape, generator=torch.Generator().manual_seed(1))
    return y, v, resize_adjoint(v, th, tw, H, W)


# (B, C, H, W, scale, antialiasing): factors 2, 3, 4, 8 with and without antialiasing, odd sizes, upscaling, sizes that put
# a tile edge on every border (16-row tiles, 64-column tiles, and the tile widths the shared-memory budget halves to)
CASES = [
    (2, 3, 23, 17, 1 / 2, True), (2, 3, 23, 17, 1 / 3, True), (1, 2, 37, 29, 1 / 4, True), (2, 1, 21, 30, 1 / 2, False),
    (1, 3, 33, 19, 1 / 4, False), (1, 1, 70, 131, 1 / 3, True), (1, 1, 65, 257, 1 / 2, True), (1, 2, 130, 66, 1 / 4, True),
    (1, 1, 300, 41, 1 / 8, True), (1, 1, 47, 140, 1 / 8, False), (1, 2, 19, 37, 2.0, True), (1, 1, 9, 33, 4.0, True),
    (1, 1, 17, 65, 1.5, True), (3, 1, 16, 64, 1 / 2, True), (1, 1, 12, 12, 1 / 1.5, True), (1, 1, 5, 6, 1 / 2, True),
]


@pytest.mark.parametrize("B,C,H,W,scale,aa", CASES)
def test_against_fp64_restatement(emul_ops, B, C, H, W, scale, aa):
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(H * W))
    y, v, xt = run(x, scale, aa)
    # the reference evaluates the tap positions (i + 0.5) / scale in fp32: exact for power-of-two scales, rounded otherwise
    tol = 1e-6 if math.log2(scale).is_integer() or scale in (1 / 3,) else 3e-6
    MH, MW = R.operators(H, W, scale, aa)
    assert rel_err(y, R.apply(x, MH, MW)) < tol
    assert rel_err(xt, R.apply_t(v, MH, MW)) < tol
    # against the same operator assembled in fp64 from the library's fp32 tables: only the kernels' own rounding remains
    TH, TW = table_matrix(H, MH.shape[0], scale, aa), table_matrix(W, MW.shape[0], scale, aa)
    assert rel_err(y, R.apply(x, TH, TW)) < 1e-6
    assert rel_err(xt, R.apply_t(v, TH, TW)) < 1e-6
    # adjointness in fp64
    lhs, rhs = float((y.double() * v.double()).sum()), float((x.double() * xt.double()).sum())
    assert abs(lhs - rhs) <= 1e-6 * (y.double().norm() * v.double().norm())


def test_sizes_mode_one_axis_identity(emul_ops):
    """sizes that keep one axis: that axis runs as a one-tap band, bitwise the input"""
    import deepinv_b200 as dinv

    x = torch.randn(2, 2, 13, 40, generator=torch.Generator().manual_seed(3))
    y = dinv.physics.functional.imresize_matlab(x, sizes=(13, 20))
    MW = R.matrix(40, 20, 0.5)
    assert rel_err(y, R.apply(x, torch.eye(13, dtype=torch.float64), MW)) < 1e-6
    assert torch.equal(dinv.physics.functional.imresize_matlab(x, sizes=(13, 40)), x)


def test_reproducible(emul_ops):
    x = torch.randn(2, 2, 45, 70, generator=torch.Generator().manual_seed(4))
    a, b = run(x, 1 / 3), run(x, 1 / 3)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])


def test_empty_batch_and_bad_arguments():
    from deepinv_b200.physics.imresize import axis_table

    lib = emul_lib()
    th, tw = axis_table(20, 10, 0.5), axis_table(30, 15, 0.5)
    x, y = torch.randn(1, 20, 30), torch.full((1, 10, 15), float("nan"))
    f = lambda BC, H=20, W=30, Ho=10, Wo=15, kw=tw.k, s=0.5, xx=x: lib.dinvk_resize_fwd(  # noqa: E731
        ptr(xx), ptr(y), BC, H, W, Ho, Wo, ptr(th.base), ptr(th.weight), th.k, ptr(tw.base), ptr(tw.weight), kw, s, None)
    n0 = lib.dinvk_launch_count()
    assert f(0) == 0 and lib.dinvk_launch_count() == n0  # empty batch: no launch
    assert f(-1) == EINVAL and b"bad shape" in lib.dinvk_last_error()
    assert f(1, Ho=0) == EINVAL
    assert f(1, kw=0) == EINVAL and b"tap" in lib.dinvk_last_error()
    assert f(1, s=0.0) == EINVAL and b"scale" in lib.dinvk_last_error()
    assert f(1, s=float("nan")) == EINVAL
    assert f(1, xx=None) == EINVAL and b"null" in lib.dinvk_last_error()
    assert f(1, kw=100000) == EUNSUPPORTED  # a band no tile width can hold
    assert lib.dinvk_launch_count() == n0
    assert f(1) == 0 and torch.isfinite(y).all()
    g = lambda BC, tab=th.ptr: lib.dinvk_resize_adj(ptr(y), ptr(x), BC, 20, 30, 10, 15, ptr(tab), ptr(th.out), ptr(th.wt),  # noqa: E731
                                                   ptr(tw.ptr), ptr(tw.out), ptr(tw.wt), tw.k, 0.5, None)
    assert g(0) == 0
    assert g(1, tab=None) == EINVAL and b"null table" in lib.dinvk_last_error()
    assert ctypes.c_int(g(1)).value == 0


# ---- the package's classes on the emulated library, against the reference's golden vectors -------------------------------
@pytest.mark.parametrize("name", golden_names("resize_f"))
def test_downsampling_matlab_golden(emul_ops, name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    p = dinv.physics.DownsamplingMatlab(factor=float(g["factor"]) if float(g["factor"]) % 1 else int(g["factor"]),
                                        antialiasing=bool(int(g["aa"])))
    assert p.factor == int(g["stored_factor"]) and p.padding == "reflect" and p.kernel == "cubic"
    assert p.max_iter == int(g["max_iter"]) and p.tol == float(g["tol"])
    assert rel_err(p.A(g["x"]), g["y"]) < 1e-5
    assert p.A_adjoint(g["v"]).shape == g["At"].shape
    assert rel_err(p.A_adjoint(g["v"]), g["At"]) < 1e-5
    with torch.no_grad():
        assert rel_err(p.A_dagger(g["y"]), g["dagger"]) < 1e-4
        if int(g["prox_err"]) >= 0:
            with pytest.raises(ERRORS[int(g["prox_err"])]):
                p.prox_l2(g["x"], g["y"], 0.5)
        else:
            assert rel_err(p.prox_l2(g["x"], g["y"], 0.5), g["prox"]) < 1e-4
        assert rel_err(p.prox_l2(g["z"], g["y"], 0.5), g["prox_even"]) < 1e-4
    # gradients: through A by the transpose kernel, through A_adjoint by the forward kernel
    x = g["x"].clone().requires_grad_()
    (gx,) = torch.autograd.grad((p.A(x) * g["y"]).sum(), x)
    if p.factor == 1:
        assert torch.equal(gx, g["y"])
    else:  # the transpose onto x's own grid, which is A_adjoint's only when H and W are multiples of the factor
        MH, MW = R.operators(*x.shape[-2:], 1 / p.factor, bool(int(g["aa"])))
        assert rel_err(gx, R.apply_t(g["y"], MH, MW)) < 1e-6
    v = g["v"].clone().requires_grad_()
    (gv,) = torch.autograd.grad((p.A_adjoint(v) * g["At"]).sum(), v)
    assert rel_err(gv, p.A(g["At"])) < 1e-6


def test_gradient_through_A_is_the_adjoint(emul_ops):
    import deepinv_b200 as dinv

    p = dinv.physics.DownsamplingMatlab(factor=3)
    x = torch.randn(2, 2, 24, 30, generator=torch.Generator().manual_seed(5)).requires_grad_()
    w = torch.randn(2, 2, 8, 10, generator=torch.Generator().manual_seed(6))
    (gx,) = torch.autograd.grad((p.A(x) * w).sum(), x)
    assert torch.equal(gx, p.A_adjoint(w))


@pytest.mark.parametrize("name", golden_names("resize_tiny_"))
def test_tiny_images_raise_like_the_reference(emul_ops, name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    with pytest.raises(ERRORS[int(g["err"])]):
        dinv.physics.DownsamplingMatlab(factor=int(g["factor"])).A(g["x"])


def test_imresize_matlab_golden(emul_ops):
    import deepinv_b200 as dinv

    F = dinv.physics.functional
    g = load_golden("resize_up2")
    assert rel_err(F.imresize_matlab(g["x"], scale=2), g["up2"]) < 1e-5
    assert rel_err(F.imresize_matlab(g["x"], scale=2, antialiasing=False), g["up2_noaa"]) < 1e-5
    assert rel_err(F.imresize_matlab(g["x"], sizes=(25, 17)), g["up_sizes"]) < 1e-5
    assert rel_err(F.imresize_matlab(g["x"], sizes=(6, 9)), g["down_sizes"]) < 1e-5
    assert rel_err(F.imresize_matlab(g["x3"], scale=2), g["up2_3d"]) < 1e-5
    with pytest.raises(ValueError):
        F.imresize_matlab(g["x"])
    with pytest.raises(ValueError):
        F.imresize_matlab(g["x"], scale=2, sizes=(4, 4))
    with pytest.raises(ValueError):
        F.imresize_matlab(g["x"][None], scale=2)
    with pytest.raises(ValueError):
        F.imresize_matlab(g["x"], scale=2, kernel="lanczos")
    with pytest.raises(ValueError):
        F.imresize_matlab(g["x"], scale=2, padding_type="circular")
    with pytest.raises(NotImplementedError):
        F.imresize_matlab(g["x"], scale=2, kernel="gaussian")


@pytest.mark.parametrize("name", [n for n in golden_names("resize_upsampling_") if n != "resize_upsampling_valid"])
def test_upsampling_golden(emul_ops, name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    pad = name.rsplit("_", 1)[1]
    u = dinv.physics.Upsampling(img_size=(3, 16, 16), filter=g["filter"], factor=2, padding=pad)
    assert rel_err(u.A(g["x"]), g["y"]) < 1e-5
    assert rel_err(u.A_adjoint(g["v"]), g["At"]) < 1e-5
    with torch.no_grad():
        if int(g["prox_err"]) >= 0:
            with pytest.raises(ERRORS[int(g["prox_err"])]):
                u.prox_l2(g["x"], g["v"], 0.5)
        else:
            assert rel_err(u.prox_l2(g["x"], g["v"], 0.5), g["prox"]) < 1e-4


def test_upsampling_valid_asserts():
    import deepinv_b200 as dinv

    assert int(load_golden("resize_upsampling_valid")["err"]) == 2
    with pytest.raises(AssertionError):
        dinv.physics.Upsampling(img_size=(3, 16, 16), filter="bicubic", padding="valid")


def test_pgd_super_resolution_golden(emul_ops):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("resize_pgd")
    p = dinv.physics.DownsamplingMatlab(factor=2)
    algo = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=float(g["stepsize"]), lambda_reg=float(g["lambda_reg"]),
               max_iter=int(g["max_iter"]), early_stop=False)
    with torch.no_grad():
        out = algo(g["y"], p)
    assert rel_err(out, g["pgd"]) < 1e-5
