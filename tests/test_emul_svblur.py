"""The space-varying blur kernels (svblur_fwd_kernel / svblur_adj_kernel in deepinv_b200/csrc/blur.cu) on the host emulation.

Checked against the reference's golden vectors (tests/golden/svblur_*.npz) and the oracle (tests/svblur_oracle.py) on
random shapes that cross the 64-pixel tile in both directions, against the emulated Blur kernels for K = 1 with w = 1
(bitwise: the same loop on the same values), on a filter large enough that the forward re-reads x for every term, and
through the package's own `SpaceVaryingBlur`, functional forms and algorithms with the emulated library behind `ops`.
"""
import pytest
import torch

import svblur_oracle as O
from conftest import golden_names, load_golden, rel_err
from emul_util import emul_lib, ptr

OPERATOR_CASES = [n for n in golden_names("svblur_") if n != "svblur_algo"]
EINVAL, EWORKSPACE, EUNSUPPORTED = 1, 2, 4


def fwd(x, w, h, pad, lib=None):
    lib = lib or emul_lib()
    x, w, h = x.float().contiguous(), w.float().contiguous(), h.float().contiguous()
    B, Cc, H, W = x.shape
    fh, fw = h.shape[-2:]
    y = torch.full((B, Cc, H - fh + 1, W - fw + 1) if pad == 0 else (B, Cc, H, W), float("nan"))
    rc = lib.dinvk_svblur_fwd(ptr(x), ptr(w), ptr(h), ptr(y), B, Cc, H, W, w.shape[0], w.shape[1], h.shape[0], h.shape[1],
                              w.shape[2], fh, fw, pad, None)
    assert rc == 0, lib.dinvk_last_error()
    return y


def adj(y, w, h, pad, H, W, lib=None):
    lib = lib or emul_lib()
    y, w, h = y.float().contiguous(), w.float().contiguous(), h.float().contiguous()
    B, Cc = y.shape[:2]
    fh, fw = h.shape[-2:]
    x = torch.full((B, Cc, H, W), float("nan"))
    nb = lib.dinvk_svblur_adj_workspace_bytes(B, Cc, H, W, fh, fw, pad)
    ws = torch.full((nb,), 255, dtype=torch.uint8)
    rc = lib.dinvk_svblur_adj(ptr(y), ptr(w), ptr(h), ptr(x), B, Cc, H, W, w.shape[0], w.shape[1], h.shape[0], h.shape[1],
                              w.shape[2], fh, fw, pad, ptr(ws), nb, None)
    assert rc == 0, lib.dinvk_last_error()
    return x


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name):
    g = load_golden(name)
    pad = int(g["pad"])
    H, W = g["x"].shape[-2:]
    assert rel_err(fwd(g["x"], g["w"], g["h"], pad), g["y"]) < 1e-5
    assert rel_err(adj(g["v"], g["w"], g["h"], pad, H, W), g["At"]) < 1e-5


@pytest.mark.parametrize("pad", range(5))
def test_random_shapes_across_tiles(pad):
    gen = torch.Generator().manual_seed(pad)
    B, Cc, H, W, K, fh, fw = 2, 2, 70, 131, 3, 9, 6
    x = torch.randn(B, Cc, H, W, generator=gen)
    w = torch.rand(1, Cc, K, H, W, generator=gen)
    h = torch.rand(B, 1, K, fh, fw, generator=gen)
    y = fwd(x, w, h, pad)
    assert rel_err(y, O.svblur_A(x, w, h, O.PADS[pad])) < 1e-5
    v = torch.randn(y.shape, generator=gen)
    xt = adj(v, w, h, pad, H, W)
    assert rel_err(xt, O.svblur_At(v, w, h, O.PADS[pad], H, W)) < 1e-5
    lhs, rhs = float((y.double() * v.double()).sum()), float((x.double() * xt.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs)


@pytest.mark.parametrize("pad", range(5))
def test_one_term_unit_multiplier_is_blur(pad):
    lib = emul_lib()
    gen = torch.Generator().manual_seed(10 + pad)
    B, Cc, H, W, fh, fw = 2, 3, 67, 70, 5, 4
    x = torch.randn(B, Cc, H, W, generator=gen)
    h = torch.rand(1, Cc, 1, fh, fw, generator=gen)
    w = torch.ones(1, 1, 1, H, W)
    y = fwd(x, w, h, pad)
    yb = torch.empty_like(y)
    assert lib.dinvk_blur_fwd(ptr(x), ptr(h), ptr(yb), B, Cc, H, W, 1, Cc, fh, fw, pad, None) == 0
    assert torch.equal(y, yb)
    xb = torch.empty(B, Cc, H, W)
    nb = lib.dinvk_blur_adj_workspace_bytes(B, Cc, H, W, fh, fw, pad)
    ws = torch.zeros(nb, dtype=torch.uint8)
    assert lib.dinvk_blur_adj(ptr(y), ptr(h), ptr(xb), B, Cc, H, W, 1, Cc, fh, fw, pad, ptr(ws), nb, None) == 0
    assert torch.equal(adj(y, w, h, pad, H, W), xb)


def test_large_filter_rereads_x():
    """84 x 84 taps: the x patch and the product patch no longer fit side by side, so the forward re-reads x per term"""
    gen = torch.Generator().manual_seed(3)
    H, W, K = 84, 100, 2
    x = torch.randn(1, 1, H, W, generator=gen)
    w = torch.rand(1, 1, K, H, W, generator=gen)
    h = torch.rand(1, 1, K, 84, 84, generator=gen)
    assert rel_err(fwd(x, w, h, 1), O.svblur_A(x, w, h, "circular")) < 1e-5


def test_argument_errors_and_empty_batch():
    lib = emul_lib()
    x, w, h, y = torch.zeros(2, 3, 16, 16), torch.zeros(2, 3, 2, 16, 16), torch.zeros(1, 1, 2, 3, 3), torch.zeros(2, 3, 16, 16)
    ws = torch.zeros(1 << 16, dtype=torch.uint8)

    def f(*args, xp=x, wp=w, hp=h, yp=y):
        return lib.dinvk_svblur_fwd(ptr(xp), ptr(wp), ptr(hp), ptr(yp), *args, None)

    def a(*args, nb=ws.numel(), wsp=ws):
        return lib.dinvk_svblur_adj(ptr(y), ptr(w), ptr(h), ptr(x), *args, ptr(wsp) if wsp is not None else None, nb, None)

    ok = (2, 3, 16, 16, 2, 3, 1, 1, 2, 3, 3)
    assert f(*ok, 1) == 0
    assert f(*ok, 1, wp=None) == EINVAL and b"null" in lib.dinvk_last_error()
    assert f(*ok, 1, xp=None) == EINVAL
    assert f(2, 3, 16, 16, 3, 3, 1, 1, 2, 3, 3, 1) == EINVAL  # multiplier batch not in {1, B}
    assert f(2, 3, 16, 16, 2, 2, 1, 1, 2, 3, 3, 1) == EINVAL  # multiplier channels not in {1, C}
    assert f(2, 3, 16, 16, 2, 3, 2, 2, 2, 3, 3, 1) == EINVAL  # filter channels not in {1, C}
    assert f(2, 3, 16, 16, 2, 3, 1, 1, 0, 3, 3, 1) == EINVAL  # K < 1
    assert f(2, 3, 16, 16, 2, 3, 1, 1, 2, 3, 3, 7) == EINVAL  # unknown padding
    assert f(2, 3, 16, 16, 2, 3, 1, 1, 2, 17, 3, 0) == EINVAL  # valid: filter taller than the image
    assert f(2, 3, 16, 16, 2, 3, 1, 1, 2, 3, 33, 3) == EINVAL  # reflect: pad >= image size
    assert f(2, 3, 16, 16, 2, 3, 1, 1, 2, 160, 160, 1) == EUNSUPPORTED and b"too large" in lib.dinvk_last_error()
    assert a(*ok, 2, nb=16) == EWORKSPACE  # replicate folds through the workspace
    assert a(*ok, 3, wsp=None, nb=0) == EWORKSPACE
    assert a(*ok, 1, wsp=None, nb=0) == 0  # circular needs none
    assert a(2, 3, 16, 16, 2, 3, 1, 1, 0, 3, 3, 1) == EINVAL
    n0 = lib.dinvk_launch_count()
    assert f(0, 3, 16, 16, 1, 3, 1, 1, 2, 3, 3, 1) == 0 and a(0, 3, 16, 16, 1, 3, 1, 1, 2, 3, 3, 3) == 0
    assert lib.dinvk_launch_count() == n0


# ---- the package on the emulated library -------------------------------------------------------------------------------
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


@pytest.mark.parametrize("name", ["svblur_reflect_7x4_k10", "svblur_valid_5x5_k3", "svblur_bcast_mB1_f1C", "svblur_generator_valid",
                                  "svblur_fft_circular"])
def test_package_class(emul_ops, name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    pad = O.PADS[int(g["pad"])]
    phys = dinv.physics.SpaceVaryingBlur(filters=g["h"], multipliers=g["w"], padding=pad, use_fft=bool(g["use_fft"]))
    assert phys.use_fft == bool(g["use_fft"]) and phys.padding == pad
    assert rel_err(phys.A(g["x"]), g["y"]) < 1e-5
    assert rel_err(phys.A_adjoint(g["v"]), g["At"]) < 1e-5
    F = dinv.physics.functional
    assert rel_err(F.product_convolution2d(g["x"], g["w"], g["h"], padding=pad), g["y"]) < 1e-5
    assert rel_err(F.product_convolution2d_adjoint(g["v"], g["w"], g["h"], padding=pad), g["At"]) < 1e-5
    # the gradient w.r.t. x runs the adjoint kernel
    x = g["x"].clone().requires_grad_()
    (gx,) = torch.autograd.grad((phys.A(x) * g["v"]).sum(), x)
    assert rel_err(gx, g["At"]) < 1e-5


def test_package_parameters_and_errors(emul_ops):
    import deepinv_b200 as dinv

    g = load_golden("svblur_circular_5x5_k3")
    x, w, h = g["x"], g["w"], g["h"]
    phys = dinv.physics.SpaceVaryingBlur()
    assert phys.filters is None and phys.padding == "valid"
    # parameters passed to A are stored
    assert rel_err(phys.A(x, filters=h, multipliers=w, padding="circular"), g["y"]) < 1e-5
    assert phys.padding == "circular" and phys.filters is h and phys.multipliers is w
    assert rel_err(phys.A_adjoint(g["v"]), g["At"]) < 1e-5
    assert {"filters", "multipliers"} <= set(dict(phys.named_buffers()))
    # more filters than multipliers: the first K are used, as the reference indexes h[:, :, k] for k < K
    more = torch.cat([h, torch.rand_like(h[:, :, :1])], 2)
    assert rel_err(phys.A(x, filters=more), g["y"]) < 1e-5
    with pytest.raises(IndexError):
        phys.A(x, filters=h[:, :, :2])
    phys.update_parameters(filters=h)
    with pytest.raises(ValueError):
        phys.A(x, padding="wrap")
    phys.padding = "circular"
    with pytest.raises(RuntimeError):
        phys.A(x[..., :-1])  # multipliers sized for another image
    with pytest.raises(ValueError):
        phys.A(x[:, :, None])  # 5-D input
    with pytest.raises(AssertionError):
        dinv.physics.functional.product_convolution2d(x, w, torch.rand(1, 3, 3, 3, 3), padding="circular")  # filter channels


def test_package_cg_prox_and_pgd(emul_ops):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("svblur_algo")
    phys = dinv.physics.SpaceVaryingBlur(filters=g["h"], multipliers=g["w"], padding=O.PADS[int(g["pad"])])
    assert phys.max_iter == int(g["max_iter"]) and phys.tol == float(g["tol"])
    with torch.no_grad():
        assert rel_err(phys.prox_l2(g["z"], g["y"], float(g["gamma"])), g["prox"]) < 1e-5
        out = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(g["y"], phys)
    assert rel_err(out, g["pgd"]) < 1e-5
