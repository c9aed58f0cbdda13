"""The property checks the reference's own physics tests make (deepinv/tests/test_physics.py: adjointness :717-745, spectral norm
:882-926, pseudo-inverse :946-968, MRI zero pattern :996-1091) for its `3DMRI` and `3DMultiCoilMRI` test operators (:184-188,
218-231, at (2, 5, 17, 11) and 15 coils of ones / sqrt(15)), re-run on the drop-in classes over the emulated kernels."""
from math import sqrt

import pytest
import torch

SHAPE = (2, 5, 17, 11)


@pytest.fixture(autouse=True)
def emul_backend(monkeypatch):
    from emul_util import emul_lib

    from deepinv_b200 import ops

    lib = emul_lib()

    def check(rc):
        assert rc == 0, lib.dinvk_last_error()

    monkeypatch.setattr(ops, "_require_cuda", lambda *ts: torch.device("cpu"))
    monkeypatch.setattr(ops, "_stream", lambda dev: None)
    monkeypatch.setattr(ops, "get_lib", lambda: lib)
    monkeypatch.setattr(ops, "check", check)
    ops._ws_cache.clear()
    yield
    ops._ws_cache.clear()


def _find_operator(name, mask=None):
    import deepinv_b200 as dinv

    P = dinv.physics
    if name == "3DMRI":
        return P.MRI(mask=mask, img_size=SHAPE, three_d=True)
    maps = torch.ones(1, 15, *SHAPE[1:], dtype=torch.complex64) / sqrt(15)
    return P.MultiCoilMRI(mask=mask, coil_maps=maps, img_size=SHAPE, three_d=True)


def _mask():
    return (torch.rand(*SHAPE[1:], generator=torch.Generator().manual_seed(0)) > 0.5).float()


@pytest.mark.parametrize("name", ["3DMRI", "3DMultiCoilMRI"])
@pytest.mark.parametrize("masked", [False, True])
def test_adjointness_and_autograd_adjoint(name, masked):
    phys = _find_operator(name, _mask() if masked else None)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, *SHAPE, generator=g)
    assert abs(complex(phys.adjointness_test(x)).real) < 1e-3
    y = phys.A(x)
    v = torch.randn(y.shape, generator=g)
    xr = x.clone().requires_grad_(True)
    (grad,) = torch.autograd.grad((phys.A(xr) * v).sum(), xr)
    ref = phys.A_adjoint(v)
    assert float((grad - ref).norm() / ref.norm()) < 1e-5


@pytest.mark.parametrize("name", ["3DMRI", "3DMultiCoilMRI"])
def test_spectral_norm_by_power_method(name):
    phys = _find_operator(name)
    x0 = torch.randn(1, *SHAPE, generator=torch.Generator().manual_seed(2))
    norm = float(phys.compute_norm(x0, max_iter=60, tol=1e-4, verbose=False))
    assert abs(norm - 1.0) < 0.05, norm


@pytest.mark.parametrize("name", ["3DMRI", "3DMultiCoilMRI"])
def test_pseudo_inverse_reproduces_the_measurements(name):
    phys = _find_operator(name, _mask())
    x = torch.randn(1, *SHAPE, generator=torch.Generator().manual_seed(3))
    r = phys.A(x)
    y = phys.A(phys.A_dagger(r))
    assert float((y - r).norm() / r.norm()) < 0.05


@pytest.mark.parametrize("name", ["3DMRI", "3DMultiCoilMRI"])
def test_mri_zero_pattern(name):
    mask = _mask()
    phys = _find_operator(name, mask)
    x = torch.randn(2, *SHAPE, generator=torch.Generator().manual_seed(4))
    y = phys.A(x)
    m = mask.bool()
    if name == "3DMultiCoilMRI":
        assert y.shape == (2, 2, 15, *SHAPE[1:])
        m = m[None, None, None]
    assert torch.all(y[(~m).expand_as(y)] == 0) and torch.all(y[m.expand_as(y)] != 0)


def test_transform_of_a_coil_stack():
    """the mixin's V / V^T with three_d=True on a (B,2,N,D,H,W) k-space: fftn over (-3,-2,-1) per coil, as the reference's
    mixin computes it (its MultiCoilMRI passes exactly this layout); a tensor of lower rank is refused"""
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent))
    import mri3d_ref64 as S

    import deepinv_b200 as dinv

    mix = dinv.physics.mri.MRIMixin()
    g = torch.Generator().manual_seed(6)
    for shape in ((1, 2, 3, 4, 6, 8), (2, 2, 2, 3, 5, 7, 6), (2, 2, 4, 6, 8)):
        y = torch.randn(*shape, generator=g)
        yc = torch.complex(y[:, 0].double(), y[:, 1].double())
        for inverse, fn in ((False, mix.im_to_kspace), (True, mix.kspace_to_im)):
            want = S.fft3(yc, inverse)
            got = fn(y, three_d=True)
            assert got.shape == y.shape
            err = float((got.double() - torch.stack([want.real, want.imag], 1)).norm() / want.abs().norm())
            assert err < 1e-5, (shape, inverse, err)
    with pytest.raises(ValueError):
        mix.im_to_kspace(torch.randn(2, 2, 6, 8), three_d=True)
    with pytest.raises(ValueError):
        mix.kspace_to_im(torch.randn(2, 3, 4, 6, 8), three_d=True)
