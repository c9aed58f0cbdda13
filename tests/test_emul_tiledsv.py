"""The tiled space-varying blur kernels (tiled_svblur_fwd_kernel / tiled_svblur_adj_kernel in deepinv_b200/csrc/blur.cu) on the
host emulation.

Checked against the reference's golden vectors (tests/golden/tiledsv_*.npz) and the oracle (tests/tiledsv_oracle.py) on random
shapes that cross the 64-pixel tile in both directions, against the emulated Blur kernel when one patch covers the image
(bitwise), for the reach of a non-finite filter, and through the package's own `TiledSpaceVaryingBlur`, generator and
algorithms with the emulated library behind `ops`.
"""
import pytest
import torch

import tiledsv_oracle as O
from conftest import golden_names, load_golden, rel_err
from emul_util import emul_lib, ptr

OPERATOR_CASES = [n for n in golden_names("tiledsv_") if n != "tiledsv_algo"]
EINVAL, EUNSUPPORTED = 1, 4


def geometry(g):
    return tuple(int(v) for v in g["patch"]), tuple(int(v) for v in g["stride"])


def fwd(x, w, h, patch, stride, lib=None):
    lib = lib or emul_lib()
    x, w, h = x.float().contiguous(), w.float().contiguous(), h.float().contiguous()
    B, Cc, H, W = x.shape
    fh, fw = h.shape[-2:]
    y = torch.full((B, Cc, H - fh + 1, W - fw + 1), float("nan"))
    rc = lib.dinvk_tiled_svblur_fwd(ptr(x), ptr(w), ptr(h), ptr(y), B, Cc, H, W, h.shape[0], h.shape[1], h.shape[2], fh, fw,
                                    *patch, *stride, None)
    assert rc == 0, lib.dinvk_last_error()
    return y


def adj(y, w, h, patch, stride, H, W, lib=None):
    lib = lib or emul_lib()
    y, w, h = y.float().contiguous(), w.float().contiguous(), h.float().contiguous()
    B, Cc = y.shape[:2]
    fh, fw = h.shape[-2:]
    x = torch.full((B, Cc, H, W), float("nan"))
    rc = lib.dinvk_tiled_svblur_adj(ptr(y), ptr(w), ptr(h), ptr(x), B, Cc, H, W, h.shape[0], h.shape[1], h.shape[2], fh, fw,
                                    *patch, *stride, None)
    assert rc == 0, lib.dinvk_last_error()
    return x


def multipliers(H, W, patch, stride, mode="bump"):
    from deepinv_b200.physics import TiledSpaceVaryingBlur
    from deepinv_b200.physics.functional import generate_tiled_multipliers

    size = TiledSpaceVaryingBlur(patch_size=patch, stride=stride).get_compatible_img_size((H, W))
    return generate_tiled_multipliers(size, patch, stride, mode)


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name):
    g = load_golden(name)
    patch, stride = geometry(g)
    H, W = g["x"].shape[-2:]
    assert rel_err(fwd(g["x"], g["w"], g["h"], patch, stride), g["y"]) < 1e-5
    assert rel_err(adj(g["v"], g["w"], g["h"], patch, stride, H, W), g["At"]) < 1e-5


@pytest.mark.parametrize("H,W,fh,fw,patch,stride", [(70, 131, 9, 6, (40, 64), (20, 64)), (130, 75, 4, 7, (64, 30), (64, 17)),
                                                    (97, 66, 31, 31, 32, 16), (300, 257, 7, 7, (100, 90), (70, 50))])
def test_random_shapes_across_tiles(H, W, fh, fw, patch, stride):
    gen = torch.Generator().manual_seed(H)
    patch, stride = (patch, patch) if isinstance(patch, int) else patch, (stride, stride) if isinstance(stride, int) else stride
    nr, nc = O.num_patches(H, W, patch, stride)
    x = torch.randn(2, 2, H, W, generator=gen)
    h = torch.rand(2, 1, nr * nc, fh, fw, generator=gen)
    w = multipliers(H, W, patch, stride)
    y = fwd(x, w, h, patch, stride)
    assert rel_err(y, O.tiledsv_A(x, w, h, patch, stride)) < 1e-5
    v = torch.randn(y.shape, generator=gen)
    xt = adj(v, w, h, patch, stride, H, W)
    assert rel_err(xt, O.tiledsv_At(v, w, h, patch, stride, H, W)) < 1e-5
    lhs, rhs = float((y.double() * v.double()).sum()), float((x.double() * xt.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs)


def test_one_patch_is_blur():
    lib = emul_lib()
    gen = torch.Generator().manual_seed(10)
    B, Cc, H, W, fh, fw = 2, 3, 67, 70, 5, 4
    x = torch.randn(B, Cc, H, W, generator=gen)
    h = torch.rand(1, Cc, 1, fh, fw, generator=gen)
    w = multipliers(H, W, (H, W), (H, W))
    assert torch.equal(w, torch.ones(1, 1, 1, H, W))
    y = fwd(x, w, h, (H, W), (H, W))
    yb = torch.empty_like(y)
    assert lib.dinvk_blur_fwd(ptr(x), ptr(h[:, :, 0].contiguous()), ptr(yb), B, Cc, H, W, 1, Cc, fh, fw, 0, None) == 0
    assert torch.equal(y, yb)
    xb = torch.empty(B, Cc, H, W)
    assert lib.dinvk_blur_adj(ptr(y), ptr(h[:, :, 0].contiguous()), ptr(xb), B, Cc, H, W, 1, Cc, fh, fw, 0, None, 0, None) == 0
    assert torch.equal(adj(y, w, h, (H, W), (H, W), H, W), xb)


@pytest.mark.parametrize("k", [0, 4, 11])
def test_nan_filter_reaches_its_patch_only(k):
    """a NaN in h_k reaches exactly patch k's footprint in y (cropped to y) and that footprint grown by the filter in A^T y"""
    H, W, fh, fw, patch, stride = 75, 70, 5, 6, (30, 28), (15, 14)
    nr, nc = O.num_patches(H, W, patch, stride)
    gen = torch.Generator().manual_seed(k)
    x = torch.randn(1, 1, H, W, generator=gen)
    h = torch.rand(1, 1, nr * nc, fh, fw, generator=gen)
    h[0, 0, k, 2, 3] = float("nan")
    w = multipliers(H, W, patch, stride)
    r, c = divmod(k, nc)
    foot = torch.zeros(H + patch[0], W + patch[1], dtype=torch.bool)
    foot[r * stride[0]: r * stride[0] + patch[0], c * stride[1]: c * stride[1] + patch[1]] = True
    yfoot = foot[fh // 2: fh // 2 + H - fh + 1, fw // 2: fw // 2 + W - fw + 1]
    y = fwd(x, w, h, patch, stride)
    assert torch.equal(torch.isnan(y[0, 0]), yfoot)
    v = torch.randn(y.shape, generator=gen)
    xt = adj(v, w, h, patch, stride, H, W)
    grown = torch.zeros(H + fh + patch[0], W + fw + patch[1], dtype=torch.bool)
    i0, j0 = r * stride[0] - fh // 2, c * stride[1] - fw // 2  # patch origin in y coordinates, then spread by the filter
    rows = slice(max(i0, 0), max(min(i0 + patch[0], H - fh + 1), 0) + fh - 1)
    cols = slice(max(j0, 0), max(min(j0 + patch[1], W - fw + 1), 0) + fw - 1)
    grown[rows, cols] = True
    assert torch.equal(torch.isnan(xt[0, 0]), grown[:H, :W])


def test_argument_errors_and_empty_batch():
    lib = emul_lib()
    x, y = torch.zeros(2, 3, 32, 32), torch.zeros(2, 3, 30, 30)
    w, h = torch.zeros(1, 1, 49, 8, 8), torch.zeros(1, 1, 49, 3, 3)

    def f(*args, xp=x, wp=w, hp=h, yp=y):
        return lib.dinvk_tiled_svblur_fwd(ptr(xp), ptr(wp), ptr(hp), ptr(yp), *args, None)

    def a(*args):
        return lib.dinvk_tiled_svblur_adj(ptr(y), ptr(w), ptr(h), ptr(x), *args, None)

    ok = (2, 3, 32, 32, 1, 1, 49, 3, 3, 8, 8, 4, 4)
    assert f(*ok) == 0 and a(*ok) == 0
    assert f(*ok, wp=None) == EINVAL and b"null" in lib.dinvk_last_error()
    assert f(*ok, xp=None) == EINVAL and f(*ok, hp=None) == EINVAL and f(*ok, yp=None) == EINVAL
    assert f(2, 3, 32, 32, 1, 1, 48, 3, 3, 8, 8, 4, 4) == EINVAL and b"patches" in lib.dinvk_last_error()  # nr * nc != K
    assert f(2, 3, 32, 32, 1, 1, 16, 3, 3, 8, 8, 9, 8) == EINVAL  # stride > patch
    assert f(2, 3, 32, 32, 1, 1, 49, 3, 3, 8, 8, 0, 4) == EINVAL
    assert f(2, 3, 32, 32, 3, 1, 49, 3, 3, 8, 8, 4, 4) == EINVAL  # filter batch not in {1, B}
    assert f(2, 3, 32, 32, 1, 2, 49, 3, 3, 8, 8, 4, 4) == EINVAL  # filter channels not in {1, C}
    assert f(2, 3, 32, 32, 1, 1, 49, 33, 3, 8, 8, 4, 4) == EINVAL  # filter taller than the image
    assert f(2, 3, 5, 32, 1, 1, 7, 3, 3, 16, 8, 8, 4) == EINVAL  # the image pads to less than one patch
    assert a(2, 3, 32, 32, 1, 1, 48, 3, 3, 8, 8, 4, 4) == EINVAL
    big = torch.zeros(1, 1, 1, 240, 240)
    assert lib.dinvk_tiled_svblur_fwd(ptr(big), ptr(big), ptr(big), ptr(big), 1, 1, 240, 240, 1, 1, 1, 230, 230, 240, 240, 240,
                                      240, None) == EUNSUPPORTED
    n0 = lib.dinvk_launch_count()
    assert f(0, 3, 32, 32, 1, 1, 49, 3, 3, 8, 8, 4, 4) == 0 and a(0, 3, 32, 32, 1, 1, 49, 3, 3, 8, 8, 4, 4) == 0
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
    yield lib


@pytest.mark.parametrize("name", ["tiledsv_reference_case", "tiledsv_grid2_linear", "tiledsv_bcast_fB1", "tiledsv_generator",
                                  "tiledsv_stride_eq_patch"])
def test_package_class(emul_ops, name):
    import deepinv_b200 as dinv

    g = load_golden(name)
    patch, stride = geometry(g)
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=g["h"], patch_size=patch, stride=stride,
                                              blending_mode=O.MODES[int(g["mode"])], use_fft=bool(g["use_fft"]))
    assert phys.use_fft == bool(g["use_fft"]) and phys.patch_size == patch and phys.stride == stride
    assert rel_err(phys.A(g["x"]), g["y"]) < 1e-5
    assert torch.equal(phys.multipliers, g["w"])
    assert rel_err(phys.A_adjoint(g["v"]), g["At"]) < 1e-5
    # the gradient w.r.t. x runs the adjoint kernel
    x = g["x"].clone().requires_grad_()
    (gx,) = torch.autograd.grad((phys.A(x) * g["v"]).sum(), x)
    assert rel_err(gx, g["At"]) < 1e-5


def test_package_parameters_and_errors(emul_ops):
    import deepinv_b200 as dinv

    g = load_golden("tiledsv_grid0_bump")
    patch, stride = geometry(g)
    phys = dinv.physics.TiledSpaceVaryingBlur(patch_size=patch, stride=stride)
    assert phys.filters is None and phys.multipliers is None and phys.blending_mode == "bump" and phys.use_fft
    # filters passed to A are stored; the multipliers follow the image size
    assert rel_err(phys.A(g["x"], filters=g["h"]), g["y"]) < 1e-5
    assert phys.filters is g["h"] and {"filters", "multipliers"} <= set(dict(phys.named_buffers()))
    w = phys.multipliers
    assert rel_err(phys.A_adjoint(g["v"]), g["At"]) < 1e-5
    assert phys.multipliers is w  # same image size: not regenerated
    with pytest.raises(ValueError, match="number of PSFs"):
        phys.A(g["x"][..., :-8])  # another image size: more patches than filters
    assert tuple(phys.multipliers.shape[-2:]) == patch
    with pytest.raises(ValueError, match="number of PSFs"):
        phys.A(g["x"], filters=g["h"][:, :, :-1])
    phys.update_parameters(filters=g["h"])
    phys.multipliers = w.expand(2, 1, *w.shape[2:])
    with pytest.raises(NotImplementedError):
        phys.A_adjoint(g["v"])
    with pytest.raises(ValueError):
        dinv.physics.TiledSpaceVaryingBlur(patch_size=8, stride=9)
    with pytest.raises(ValueError):
        dinv.physics.TiledSpaceVaryingBlur(filters=g["h"], patch_size=patch, stride=stride, blending_mode="cosine").A(g["x"])
    with pytest.raises(ZeroDivisionError):
        dinv.physics.TiledSpaceVaryingBlur(filters=g["h"][:, :, :16], patch_size=8, stride=8, blending_mode="linear").A(g["x"])
    T = dinv.physics.TiledSpaceVaryingBlur
    assert T.num_filters((32, 33), (8, 9), (4, 5)) == O.num_patches(32, 33, (8, 9), (4, 5))
    assert phys.get_needed_pad((33, 33)) == (3, 3) and phys.get_compatible_img_size((33, 33)) == (36, 36)


def test_generator_reproduces_reference():
    import deepinv_b200 as dinv

    g = load_golden("tiledsv_generator")
    gen = dinv.physics.generator.TiledBlurGenerator(dinv.physics.generator.MotionBlurGenerator((9, 9)), patch_size=(24, 20),
                                                    stride=(12, 10))
    h = gen.step(batch_size=2, img_size=(70, 64), seed=5)["filters"]
    assert h.shape == g["h"].shape and rel_err(h, g["h"]) < 1e-6


def test_package_cg_prox_and_pgd(emul_ops):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, Tikhonov

    g = load_golden("tiledsv_algo")
    patch, stride = geometry(g)
    phys = dinv.physics.TiledSpaceVaryingBlur(filters=g["h"], patch_size=patch, stride=stride)
    assert phys.max_iter == int(g["max_iter"]) and phys.tol == float(g["tol"])
    with torch.no_grad():
        assert rel_err(phys.prox_l2(g["z"], g["y"], float(g["gamma"])), g["prox"]) < 1e-5
        out = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(g["y"], phys)
    assert rel_err(out, g["pgd"]) < 1e-5
