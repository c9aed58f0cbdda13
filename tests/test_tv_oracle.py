"""The TV oracle (tests/tv_oracle.py) against the real reference's outputs recorded in tests/golden/tv_*.npz."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tv_oracle as O  # noqa: E402
from conftest import golden_names, load_golden, rel_err  # noqa: E402

DENOISER_CASES = [n for n in golden_names("tv_") if n.startswith(("tv_iso", "tv_l1"))]


def _ths(z):
    return z["ths"] if z["ths"].dim() else float(z["ths"])


def test_fixtures_exist():
    assert len(DENOISER_CASES) >= 6 and "tv_prior" in golden_names("tv_") and "tv_algo_blur" in golden_names("tv_")


@pytest.mark.parametrize("name", DENOISER_CASES)
def test_oracle_denoiser_and_warm_restart(name):
    z = load_golden(name)
    kw = dict(l1=bool(z["l1"]), n_it_max=int(z["n_it_max"]), crit=float(z["crit"]))
    x1, u1, n1, _ = O.tv_denoise(z["y"], _ths(z), **kw)
    assert n1 == int(z["n_iter1"])
    assert torch.equal(x1, z["out1"])
    assert torch.equal(torch.isnan(u1), torch.isnan(z["u2_1"]))
    assert torch.equal(torch.nan_to_num(u1), torch.nan_to_num(z["u2_1"]))
    x2, u2, n2, _ = O.tv_denoise(z["y2"], _ths(z), x2=x1, u2=u1, **kw)
    assert n2 == int(z["n_iter2"])
    assert torch.equal(x2, z["out2"])


def test_ths_zero_is_the_identity():
    z = load_golden("tv_iso_ths0")
    assert rel_err(z["out1"], z["y"]) < 1e-6


def test_oracle_prior_functions():
    z = load_golden("tv_prior")
    assert torch.equal(O.tv_nabla(z["x"]), z["nabla"])
    assert torch.equal(O.tv_nabla_adjoint(z["gfield"]), z["nabla_adjoint"])
    assert torch.equal(O.tv_grad(z["x"]), z["grad"])
    assert rel_err(O.tv_fn(z["x"]), z["fn"]) < 1e-6
    assert rel_err(O.tv_fn(z["x"], l1=True), z["fn_l1"]) < 1e-6
