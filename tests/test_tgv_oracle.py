"""The TGV oracle (tests/tgv_oracle.py) against the real reference's outputs recorded in tests/golden/tgv_*.npz."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tgv_oracle as O  # noqa: E402
from conftest import golden_names, load_golden  # noqa: E402

DENOISER_CASES = [n for n in golden_names("tgv_") if n not in ("tgv_stencils", "tgv_algo_blur")]


def _ths(z):
    return z["ths"] if z["ths"].dim() else float(z["ths"])


def _same(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.nan_to_num(a), torch.nan_to_num(b))


def test_fixtures_exist():
    assert len(DENOISER_CASES) >= 5 and {"tgv_stencils", "tgv_algo_blur"} <= set(golden_names("tgv_"))


@pytest.mark.parametrize("name", DENOISER_CASES)
def test_oracle_denoiser_and_warm_restart_bitwise(name):
    z = load_golden(name)
    kw = dict(n_it_max=int(z["n_it_max"]), crit=float(z["crit"]))
    x1, r1, u1, n1, _ = O.tgv_denoise(z["y"], _ths(z), **kw)
    assert n1 == int(z["n_iter1"])
    assert _same(x1, z["out1"]) and _same(r1, z["r2_1"]) and _same(u1, z["u2_1"])
    x2, r2, u2, n2, _ = O.tgv_denoise(z["y2"], _ths(z), x2=x1, r2=r1, u2=u1, **kw)
    assert n2 == int(z["n_iter2"])
    assert _same(x2, z["out2"]) and _same(r2, z["r2_2"]) and _same(u2, z["u2_2"])


def test_early_break_lands_inside_a_launch():
    """for 2 and 4 iterations per launch alike: the kernel has to replay the break"""
    z = load_golden("tgv_early")
    assert int(z["converged1"]) == 1 and int(z["n_iter1"]) % 2 == 1


def test_ths_zero_is_all_nan():
    z = load_golden("tgv_ths0")
    assert torch.isnan(z["out1"]).all() and torch.isnan(z["out2"]).all()


def test_oracle_stencils_bitwise():
    z = load_golden("tgv_stencils")
    assert torch.equal(O.tgv_epsilon(z["f"]), z["epsilon"])
    assert torch.equal(O.tgv_epsilon_adjoint(z["gfield"]), z["epsilon_adjoint"])


def test_last_axis_sums_run_left_to_right():
    """torch's CPU sum over a last axis of 4 (2) rounds as ((a + b) + c) + d (a + b): the oracle writes that order out,
    and pairwise (a + b) + (c + d) differs from torch on some rows"""
    g = torch.Generator().manual_seed(0)
    v = torch.randn(1 << 16, 4, generator=g) * torch.logspace(-3, 3, 4)
    sq = v * v
    torch_sum = torch.sum(v ** 2, dim=-1)
    assert torch.equal(O._sq_sum_last(v), torch_sum)
    assert torch.equal(((sq[:, 0] + sq[:, 1]) + sq[:, 2]) + sq[:, 3], torch_sum)
    assert not torch.equal((sq[:, 0] + sq[:, 1]) + (sq[:, 2] + sq[:, 3]), torch_sum)
    assert torch.equal(O._sq_sum_last(v[:, :2]), torch.sum(v[:, :2] ** 2, dim=-1))
