"""The drunet3d_* golden fixtures (deepinv v0.4.1's DRUNet(dim=3), tests/golden/make_golden_drunet3d.py) against the fp64
restatement tests/drunet3d_ref64.py (CPU) and against `DRUNet(dim=3)` at fp32 / tc32 / tc32h on the H100, including PnP-PGD on
`MRI(three_d=True)` and on a 3-D circular `Blur`."""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from drunet3d_ref64 import drunet3d_ref64, fixture_weights

GOLD = Path(__file__).resolve().parent / "golden"
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")


def load(name):
    with np.load(GOLD / f"{name}.npz") as f:
        return {k: f[k] for k in f.files}


def t(a):
    return torch.from_numpy(np.asarray(a))


def ref_pad(x, sigma, sd):
    """the reference's forward: test_pad (replicate to a multiple of 16) for unsafe shapes"""
    pad = [(-d) % 16 if (d % 8 or d < 32) else 0 for d in x.shape[2:]]
    if not any(pad):
        return drunet3d_ref64(x, sigma, sd, nb=1)
    pad = [(-d) % 16 for d in x.shape[2:]]
    padding = (0, pad[2], 0, pad[1], 0, pad[0])
    if torch.is_tensor(sigma) and sigma.dim() == 5 and sigma.shape[2:] == x.shape[2:]:
        sigma = F.pad(sigma, padding, mode="replicate")
    return drunet3d_ref64(F.pad(x, padding, mode="replicate"), sigma, sd, nb=1)[..., :x.shape[2], :x.shape[3], :x.shape[4]]


@pytest.mark.parametrize("name,sig", [("drunet3d_safe", "sigma"), ("drunet3d_safe", "sigma5"), ("drunet3d_pad_c1", "sigma"),
                                      ("drunet3d_pad_map", "sigma")])
def test_restatement_matches_the_reference(name, sig):
    fx = load(name)
    sd = fixture_weights(fx)
    s = fx[sig]
    out = ref_pad(t(fx["x"]), t(s) if s.ndim else float(s), sd)
    assert rel_err(out, t(fx["out5" if sig == "sigma5" else "out"])) < 1e-5


def test_state_dict_names_shapes_and_errors():
    import deepinv_b200 as dinv

    fx = load("drunet3d_safe")
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, nc=(64, 64, 128, 128), nb=1, pretrained=None, dim=3).eval()
    sd = fixture_weights(fx)
    assert sorted(m.state_dict()) == sorted(sd)
    assert all(tuple(m.state_dict()[k].shape) == tuple(v.shape) for k, v in sd.items())
    m.load_state_dict(sd, strict=True)
    x = t(fx["x"])
    with torch.no_grad():
        for key, call in (("err_sigma4", lambda: m(x, torch.ones(1, 1, 1, 1))),
                          ("err_onesplit", lambda: m(torch.zeros(1, 2, 64, 70, 66), 0.05)),
                          ("err_dim", lambda: dinv.models.DRUNet(pretrained=None, dim=4))):
            with pytest.raises(Exception) as e:
                call()
            assert type(e.value).__name__ == ERRORS[int(fx[key])], key


# ---- on the H100 ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _model(fx, ch, precision, dev):
    import deepinv_b200 as dinv

    m = dinv.models.DRUNet(in_channels=ch, out_channels=ch, nc=(64, 64, 128, 128), nb=1, pretrained=None, dim=3, precision=precision)
    m.load_state_dict(fixture_weights(fx), strict=True)
    return m.to(dev).eval()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tc32", "tc32h"])
@pytest.mark.parametrize("name", ["drunet3d_safe", "drunet3d_pad_c1", "drunet3d_pad_map"])
def test_drunet3d_vs_golden(name, precision, dev):
    fx = load(name)
    x = t(fx["x"]).to(dev)
    m = _model(fx, x.shape[1], precision, dev)
    s = fx["sigma"]
    with torch.no_grad():
        assert rel_err(m(x, t(s).to(dev) if s.ndim else float(s)), t(fx["out"])) < 1e-5
        if "sigma5" in fx:
            assert rel_err(m(x, t(fx["sigma5"]).to(dev)), t(fx["out5"])) < 1e-5


@pytest.mark.gpu
def test_pnp_pgd_mri3d_vs_golden(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP

    fx = load("drunet3d_pgd_mri")
    D, H, W = fx["mask"].shape
    phys = dinv.physics.MRI(mask=t(fx["mask"]).to(dev), img_size=(2, D, H, W), three_d=True, device=dev)
    den = _model(fx, 2, "tc32h", dev)
    with torch.no_grad():
        out = PGD(data_fidelity=L2(), prior=PnP(den), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)(t(fx["y"]).to(dev), phys)
    assert rel_err(out, t(fx["out"])) < 1e-5


@pytest.mark.gpu
def test_pnp_pgd_blur3d_vs_golden(dev):
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP

    fx = load("drunet3d_pgd_blur")
    phys = dinv.physics.Blur(filter=t(fx["filt"]).to(dev), padding="circular", device=dev)
    den = _model(fx, 1, "tc32h", dev)
    with torch.no_grad():
        out = PGD(data_fidelity=L2(), prior=PnP(den), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)(t(fx["y"]).to(dev), phys)
    assert rel_err(out, t(fx["out"])) < 1e-5
