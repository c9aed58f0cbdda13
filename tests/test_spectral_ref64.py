"""The fp64 contract of `dinvk_spectral` (tests/spectral_ref64.py) against the oracle's MRI / MultiCoilMRI / BlurFFT (oracle/ref_ops.py)
evaluated in float64: the same numbers, reached through the C ABI's arguments instead of the reference's classes."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import spectral_ref64 as S  # noqa: E402
from conftest import rel_err  # noqa: E402

TOL = 1e-12
SIZES = [(2, 12, 10), (1, 9, 7), (3, 16, 15)]


def _masks(B, H, W, g):
    """(name, (B|1,2,H,W) mask as the reference stores it, its ABI form (tensor, strides)) for full, shared, line and weighted masks"""
    full = (torch.rand(B, 2, H, W, generator=g, dtype=torch.float64) > 0.5).double()
    line = (torch.rand(B, 1, 1, W, generator=g, dtype=torch.float64) > 0.5).double()
    w = torch.rand(B, 2, H, W, generator=g, dtype=torch.float64) * (torch.rand(B, 2, H, W, generator=g, dtype=torch.float64) > 0.3)
    w.view(-1)[::7] = 3e-6  # below the pseudo-inverse threshold
    return [("full", full, (full, (2 * H * W, H * W, W))),
            ("shared", full[:1], (full[:1].contiguous(), (0, H * W, W))),
            ("line", line.expand(B, 2, H, W), (line.contiguous(), (W, 0, 0))),
            ("weighted", w, (w, (2 * H * W, H * W, W)))]


@pytest.mark.parametrize("B,H,W", SIZES)
@pytest.mark.parametrize("centered", [True, False])
def test_mri_operators(B, H, W, centered):
    from oracle import ref_ops as R

    if not centered:  # the reference's MRI is always centred: check the plain transform against torch directly
        g = torch.Generator().manual_seed(1)
        x = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
        want = R.from_complex(torch.fft.fftn(R.to_complex(x), dim=(-2, -1), norm="ortho"))
        assert rel_err(S.spectral_ref(x, H, W, fwd=True, inv=False, centered=False), want) < TOL
        want = R.from_complex(torch.fft.ifftn(R.to_complex(x), dim=(-2, -1), norm="ortho"))
        assert rel_err(S.spectral_ref(x, H, W, fwd=False, inv=True, centered=False), want) < TOL
        return
    g = torch.Generator().manual_seed(B * 100 + H * 10 + W)
    x = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    z = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    for name, m, (mt, st) in _masks(B, H, W, g):
        kw = dict(mask=mt, strides=st)
        y = R.mri_A(x, m)
        assert rel_err(S.spectral_ref(x, H, W, fwd=True, inv=False, gmode=S.G_MASK, **kw), y) < TOL, name
        assert rel_err(S.spectral_ref(y, H, W, fwd=False, inv=True, gmode=S.G_MASK, **kw), R.mri_At(y, m)) < TOL, name
        assert rel_err(S.spectral_ref(x, H, W, fwd=True, inv=True, gmode=S.G_SQ, **kw), R.mri_AtA(x, m)) < TOL, name
        assert rel_err(S.spectral_ref(y, H, W, fwd=False, inv=True, gmode=S.G_PINV, **kw), R.mri_dagger(y, m)) < TOL, name
        gamma = 0.7
        aty = S.spectral_ref(y, H, W, fwd=False, inv=True, gmode=S.G_MASK, **kw)
        prox = S.spectral_ref(aty, H, W, fwd=True, inv=True, gmode=S.G_INV_SQ_PLUS_C, p1=z, a1=1 / gamma, c=1 / gamma, **kw)
        assert rel_err(prox, R.mri_prox_l2(z, y, m, gamma)) < TOL, name
        # per-image constants override c
        cb = torch.full((B,), 1 / gamma, dtype=torch.float64)
        prox_cb = S.spectral_ref(aty, H, W, fwd=True, inv=True, gmode=S.G_INV_SQ_PLUS_C, p1=z, a1=1 / gamma, c=123.0, c_batch=cb, **kw)
        assert rel_err(prox_cb, prox) < TOL, name
        # the fused PGD data step: x - s (A^T A x - A^T y) as prologue / epilogue terms
        step = S.spectral_ref(x, H, W, fwd=True, inv=True, gmode=S.G_SQ, e0=-0.9, q0=x, e1=1.0, q1=aty, e2=0.9, **kw)
        assert rel_err(step, x - 0.9 * (R.mri_AtA(x, m) - aty)) < TOL, name
    # elementwise only: g(mask) (.) u with no transform
    mt, st = _masks(B, H, W, g)[0][2]
    assert rel_err(S.spectral_ref(x, H, W, fwd=False, inv=False, gmode=S.G_MASK, mask=mt, strides=st), mt * x) < TOL


@pytest.mark.parametrize("B,H,W", SIZES)
@pytest.mark.parametrize("shared", [True, False])
def test_multicoil(B, H, W, shared):
    from oracle import ref_ops as R

    N = 3
    g = torch.Generator().manual_seed(B + H + W + shared)
    x = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    maps = torch.randn(1 if shared else B, N, H, W, generator=g, dtype=torch.complex128)
    m = (torch.rand(B, 1, 1, W, generator=g, dtype=torch.float64) > 0.4).double().expand(B, 2, H, W).contiguous()
    kw = dict(gmode=S.G_MASK, mask=m, strides=(2 * H * W, H * W, W), ncoil=N, coil_maps=maps)
    y = R.mcmri_A(x, m, maps)
    got = S.spectral_ref(x, H, W, fwd=True, inv=False, coil_mode=1, **kw)
    assert got.shape == y.shape and rel_err(got, y) < TOL
    assert rel_err(S.spectral_ref(y, H, W, fwd=False, inv=True, coil_mode=2, **kw), R.mcmri_At(y, m, maps)) < TOL
    assert rel_err(S.spectral_ref(y, H, W, fwd=False, inv=True, coil_mode=3, **kw), R.mcmri_At(y, m, maps, use_rss=True)) < TOL
    # e0 scales the coil-combined adjoint; the rss magnitude takes no epilogue
    assert rel_err(S.spectral_ref(y, H, W, fwd=False, inv=True, coil_mode=2, e0=-0.5, **kw), -0.5 * R.mcmri_At(y, m, maps)) < TOL


def blurfft_multipliers(filt, C, H, W):
    """complex multiplier h: the full spectrum of the zero-padded, centre-rolled filter, one per (B|1, C) image, float64"""
    from oracle import ref_ops as R

    f = filt.double()
    if C > f.shape[1]:
        f = f.repeat(1, C, 1, 1)
    h = R.filter_fft(f, (C, H, W), real_fft=False)
    return h.reshape(-1, H, W)


@pytest.mark.parametrize("H,W", [(12, 10), (9, 7), (16, 15)])
@pytest.mark.parametrize("per_image", [False, True])
def test_blurfft(H, W, per_image):
    """BlurFFT as complex images with a zero imaginary plane, one complex multiplier per image (CMUL / CMUL_CONJ)"""
    from oracle import ref_ops as R

    B, C = 2, 3
    g = torch.Generator().manual_seed(H * W + per_image)
    filt = torch.rand(B if per_image else 1, C if per_image else 1, 4, 3, generator=g, dtype=torch.float64)
    filt[..., 1, 1] += 2.0  # spectrum bounded away from zero
    filt = filt / filt.sum((-2, -1), keepdim=True)
    x = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    z = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    mask, angle = R.blurfft_params(filt, (C, H, W))
    h = blurfft_multipliers(filt, C, H, W)
    if not per_image:
        h = h.repeat(B, 1, 1)  # one multiplier per image, b-major like the (B, C) batch
    hr = torch.view_as_real(h.contiguous()).contiguous()
    st = (H * W, 0, W)
    planar = lambda t: torch.stack([t.reshape(B * C, H, W), torch.zeros(B * C, H, W, dtype=torch.float64)], 1)
    real = lambda t: t[:, 0].reshape(B, C, H, W)
    run = lambda t, gm, mt, **kw: real(S.spectral_ref(planar(t), H, W, fwd=True, inv=True, centered=False, gmode=gm, mask=mt, strides=st, **kw))
    y = R.blurfft_A(x, mask, angle, (C, H, W))
    assert rel_err(run(x, S.G_CMUL, hr), y) < TOL
    aty = run(y, S.G_CMUL_CONJ, hr)
    assert rel_err(aty, R.blurfft_At(y, mask, angle, (C, H, W))) < TOL
    habs = h.abs().contiguous()
    prox = real(S.spectral_ref(planar(aty), H, W, fwd=True, inv=True, centered=False, gmode=S.G_INV_SQ_PLUS_C, mask=habs,
                               strides=st, p1=planar(z), a1=1 / 0.7, c=1 / 0.7))
    assert rel_err(prox, R.blurfft_prox_l2(z, y, mask, angle, (C, H, W), 0.7)) < TOL
    hdag = torch.where(h.abs() > 1e-5, 1 / h, torch.zeros_like(h))
    assert rel_err(run(y, S.G_CMUL, torch.view_as_real(hdag.contiguous()).contiguous()), R.blurfft_dagger(y, mask, angle, (C, H, W))) < TOL


def test_multiplier_addressing():
    """flat-memory addressing: a strided multiplier read through (sb, sc, sh), the CMUL pairs through (sb, sh) with sc ignored"""
    H, W = 3, 5
    t = torch.arange(200, dtype=torch.float64)
    g0, g1 = S.multiplier(t, S.G_MASK, 2, H, W, (40, 7, 9))
    assert g0[1, 2, 3] == 40 + 18 + 3 and g1[1, 2, 3] == 40 + 7 + 18 + 3
    m = S.multiplier(t, S.G_CMUL, 2, H, W, (20, 99, 6))
    i = 20 + 12 + 3
    assert m[1, 2, 3] == complex(2 * i, 2 * i + 1)
    assert S.multiplier(t, S.G_CMUL_CONJ, 2, H, W, (20, 99, 6))[1, 2, 3] == complex(2 * i, -(2 * i + 1))
    p0, p1 = S.multiplier(torch.tensor([0.0, 3e-6, 1e-5, 0.5, 4.0]), S.G_PINV, 1, 1, 5, (0, 0, 0))
    assert p0.reshape(-1).tolist() == [0.0, 0.0, 0.0, 2.0, 0.25]
