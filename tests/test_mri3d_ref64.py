"""The fp64 contract of `dinvk_spectral3d` (tests/mri3d_ref64.py) against the oracle's 3-D transform (oracle/ref_ops.py) in float64
and against the mri3d_* golden vectors of the real reference: the same numbers, reached through the C ABI's arguments."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import mri3d_ref64 as S  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

TOL = 1e-12
GOLD = 2e-6  # the fixtures are the reference's fp32 evaluation
MC_CASES = golden_names("mri3d_mc_")
SC_CASES = golden_names("mri3d_sc_")


def _maps(g):
    return torch.complex(g["maps_re"], g["maps_im"])


def ref_mask5(m):
    """the reference's MRI stores a (D,H,W) mask as (1,D,H,W), broadcast over batch and planes: as (1,2,D,H,W)"""
    return m.unsqueeze(1).expand(m.shape[0], 2, *m.shape[1:]).contiguous() if m.dim() == 4 else m


@pytest.mark.parametrize("dims", [(5, 17, 11), (4, 6, 8), (3, 9, 10)])
def test_transform_and_single_coil_operators(dims):
    from oracle import ref_ops as R

    g = torch.Generator().manual_seed(sum(dims))
    x = torch.randn(2, 2, *dims, generator=g, dtype=torch.float64)
    z = torch.randn(2, 2, *dims, generator=g, dtype=torch.float64)
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=False), R.im_to_kspace3(x)) < TOL
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=False, inv=True), R.kspace_to_im3(x)) < TOL
    plain = R.from_complex(torch.fft.fftn(R.to_complex(x), dim=(-3, -2, -1), norm="ortho"))
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=False, centered=False), plain) < TOL
    m = (torch.rand(2, 1, *dims, generator=g, dtype=torch.float64) > 0.5).double().expand(2, 2, *dims).contiguous()
    mt, st = S.full_mask(m)
    y = m * R.im_to_kspace3(x)
    kw = dict(gmode=S.G_MASK, mask=mt, strides=st)
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=False, **kw), y) < TOL
    aty = R.kspace_to_im3(m * y)
    assert rel_err(S.spectral3d_ref(y, *dims, fwd=False, inv=True, **kw), aty) < TOL
    kw2 = dict(mask=mt, strides=st)
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=True, gmode=S.G_SQ, **kw2), R.kspace_to_im3(m * m * R.im_to_kspace3(x))) < TOL
    gamma = 0.7
    want = R.kspace_to_im3(R.im_to_kspace3(aty + z / gamma) / (m * m + 1 / gamma))
    got = S.spectral3d_ref(aty, *dims, fwd=True, inv=True, gmode=S.G_INV_SQ_PLUS_C, p1=z, a1=1 / gamma, c=1 / gamma, **kw2)
    assert rel_err(got, want) < TOL
    cb = torch.full((2,), 1 / gamma, dtype=torch.float64)
    got = S.spectral3d_ref(aty, *dims, fwd=True, inv=True, gmode=S.G_INV_SQ_PLUS_C, p1=z, a1=1 / gamma, c=9.0, c_batch=cb, **kw2)
    assert rel_err(got, want) < TOL
    # the shared (batch-1) mask broadcasts
    mt1, st1 = S.full_mask(m[:1])
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=False, gmode=S.G_MASK, mask=mt1, strides=st1), m[:1] * R.im_to_kspace3(x)) < TOL


def test_multicoil_against_the_definition():
    """A = M F3 S_n, A^T = sum_n conj(S_n) F3^-1 M, rss = sqrt(sum |F3^-1 M y_n|^2), written out coil by coil"""
    from oracle import ref_ops as R

    g = torch.Generator().manual_seed(5)
    dims = (4, 6, 5)
    for nb, N in ((1, 3), (2, 3), (2, 1)):
        x = torch.randn(2, 2, *dims, generator=g, dtype=torch.float64)
        maps = torch.randn(nb, N, *dims, generator=g, dtype=torch.complex128)
        m = (torch.rand(2, 2, *dims, generator=g, dtype=torch.float64) > 0.4).double()
        y = S.mc_A(x, m, maps)
        xc = R.to_complex(x)
        for n in range(N):
            want = m * R.from_complex(R.cfft3(maps[:, n] * xc))
            assert rel_err(y[:, :, n], want) < TOL
        at = S.mc_At(y, m, maps)
        v = R.cfft3(R.to_complex(m[:, :, None] * y), inverse=True)
        assert rel_err(at, R.from_complex((maps.conj() * v).sum(1))) < TOL
        assert rel_err(S.mc_At(y, m, maps, rss=True), v.abs().pow(2).sum(1, keepdim=True).sqrt()) < TOL
        # adjointness
        assert abs(float((y * y).sum()) - float((x * at).sum())) < 1e-9 * float((y * y).sum())


@pytest.mark.parametrize("name", MC_CASES)
def test_multicoil_golden(name):
    g = load_golden(name)
    if "pgd" in g:
        return  # an algorithm run: checked through the package API (tests/test_gpu_mri3d.py)
    maps, mask = _maps(g), g["mask"].double()
    x, y = g["x"].double(), g["y"].double()
    assert rel_err(S.mc_A(x, mask, maps), g["y"]) < GOLD
    assert rel_err(S.mc_At(y, mask, maps), g["At"]) < GOLD


@pytest.mark.parametrize("name", SC_CASES)
def test_single_coil_golden(name):
    g = load_golden(name)
    mt, st = S.full_mask(ref_mask5(g["mask"].double()))
    dims = tuple(g["x"].shape[-3:])
    x, y, z, gamma = g["x"].double(), g["y"].double(), g["z"].double(), float(g["gamma"])
    kw = dict(mask=mt, strides=st)
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=False, gmode=S.G_MASK, **kw), g["y"]) < GOLD
    aty = S.spectral3d_ref(y, *dims, fwd=False, inv=True, gmode=S.G_MASK, **kw)
    assert rel_err(aty, g["At"]) < GOLD
    assert rel_err(S.spectral3d_ref(x, *dims, fwd=True, inv=True, gmode=S.G_SQ, **kw), g["AtA"]) < GOLD
    assert rel_err(S.spectral3d_ref(y, *dims, fwd=False, inv=True, gmode=S.G_PINV, **kw), g["dagger"]) < GOLD
    prox = S.spectral3d_ref(aty, *dims, fwd=True, inv=True, gmode=S.G_INV_SQ_PLUS_C, p1=z, a1=1 / gamma, c=1 / gamma, **kw)
    assert rel_err(prox, g["prox"]) < GOLD
