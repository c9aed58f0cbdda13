"""Pin the fp64 restatement of the Radon-family contracts (tests/radon_ref64.py) on the oracle (oracle/ref_ops.py) evaluated in
float64 and on the reference's own vectors (tests/golden/tomo_*, fan_*).  CPU only.

Also records the bound the tiled transpose's fixed-point accumulator rests on (csrc/radon.cu): at one angle, the bilinear weights
that the rotated sample lattice gives one pixel sum to between 0.83 and 1 + 4 (1 - 1/sqrt(2))^2 = 1.343, never to 2."""
import math

import numpy as np
import pytest
import torch

import radon_ref64 as RR
from conftest import golden_names, load_golden, rel_err
from oracle import ref_ops as R

TOL64 = 1e-12   # two fp64 evaluations of the same sums
TOL_GOLD = 1e-5  # the reference's fp32 results


def _am(y):
    return y.transpose(-2, -1)


@pytest.mark.parametrize("W,nang,circle", [(16, 7, False), (21, 5, True), (24, 9, False), (13, 4, False)])
def test_parallel_vs_oracle64(W, nang, circle):
    g = torch.Generator().manual_seed(W * 31 + nang)
    x = torch.randn(2, 1, W, W, generator=g, dtype=torch.float64)
    ang = torch.cat([R.default_angles(nang - 1), torch.tensor([-37.25])])
    y_ref = R.radon_forward(x, ang.double(), circle)
    assert rel_err(_am(RR.radon_fwd(x, ang, circle)), y_ref) < TOL64
    v = torch.randn(*y_ref.shape, generator=g, dtype=torch.float64)
    assert rel_err(RR.radon_adj(_am(v), ang, W, circle), R.radon_adjoint(v, ang.double(), W, circle)) < TOL64
    ir = R.iradon_backproject(v, ang.double(), W, circle) * (2 * nang) / math.pi
    assert rel_err(RR.iradon_bp(_am(v), ang, W, circle), ir) < TOL64


def test_adjoint_identity64():
    g = torch.Generator().manual_seed(3)
    for W, circle in ((30, False), (27, True)):
        ang = torch.tensor([0.0, 45.0, 90.0, 13.7, -100.0, 200.0])
        x = torch.randn(1, 2, W, W, generator=g, dtype=torch.float64)
        y = RR.radon_fwd(x, ang, circle)
        v = torch.randn(*y.shape, generator=g, dtype=torch.float64)
        lhs, rhs = float((y * v).sum()), float((x * RR.radon_adj(v, ang, W, circle)).sum())
        assert abs(lhs - rhs) <= 1e-13 * abs(lhs)
        fp = {"n_detector_pixels": 41}
        y = RR.fanbeam_fwd(x, ang, circle, fp)
        v = torch.randn(*y.shape, generator=g, dtype=torch.float64)
        lhs, rhs = float((y * v).sum()), float((x * RR.fanbeam_adj(v, ang, W, circle, fp)).sum())
        assert abs(lhs - rhs) <= 1e-13 * abs(lhs)


@pytest.mark.parametrize("W,circle,fp", [(16, False, None), (15, True, {"n_detector_pixels": 23, "detector_spacing": 0.31,
                                                                        "source_radius": 40.0, "detector_radius": 25.0})])
def test_fanbeam_vs_oracle64(W, circle, fp):
    g = torch.Generator().manual_seed(W)
    x = torch.randn(1, 2, W, W, generator=g, dtype=torch.float64)
    ang = torch.tensor([0.0, 20.0, 90.0, 133.3, 271.0])
    y_ref = R.fanbeam_forward(x, ang.double(), circle, fp)
    assert rel_err(_am(RR.fanbeam_fwd(x, ang, circle, fp)), y_ref) < TOL64
    v = torch.randn(*y_ref.shape, generator=g, dtype=torch.float64)
    assert rel_err(RR.fanbeam_adj(_am(v), ang, W, circle, fp), R.fanbeam_adjoint(v, ang.double(), W, circle, fp)) < TOL64


@pytest.mark.parametrize("N", [1, 2, 3, 8, 33, 100, 257])
def test_ramp_vs_oracle64(N):
    g = torch.Generator().manual_seed(N)
    y = torch.randn(1, 2, N, 3, generator=g, dtype=torch.float64) + 5.0
    assert rel_err(_am(RR.ramp(_am(y))), R.ramp_filter(y)) < TOL64


def test_ramp_closed_form_small():
    """the spatial sum written out: N = 4"""
    x = np.array([1.0, -2.0, 0.5, 3.0])
    k = lambda d: 0.5 if d == 0 else (-2 / (math.pi * d) ** 2 if d % 2 else 0.0)
    want = [sum(k(n - m) * x[m] for m in range(4)) for n in range(4)]
    assert np.allclose(RR.ramp(torch.tensor(x)).numpy(), want, rtol=0, atol=1e-15)


@pytest.mark.parametrize("name", [n for n in golden_names("tomo_") if "norm" not in n])
def test_tomography_golden(name):
    g = load_golden(name)
    circle = "circle" in name
    x, ang, y, v = g["x"], g["angles"], g["y"], g["v"]
    W = x.shape[-1]
    assert rel_err(_am(RR.radon_fwd(x, ang, circle)), y) < TOL_GOLD
    assert rel_err(RR.radon_adj(_am(v), ang, W, circle), g["At"]) < TOL_GOLD
    assert rel_err(RR.iradon_bp(_am(v), ang, W, circle), g["At_irad"]) < TOL_GOLD
    assert rel_err(_am(RR.ramp(_am(y))), g["filt"]) < TOL_GOLD
    n = len(ang)
    fbp = RR.radon_adj(RR.ramp(_am(y)), ang, W, circle, math.pi / (2 * n))
    assert rel_err(fbp, g["fbp"]) < TOL_GOLD
    assert rel_err(RR.iradon_bp(RR.ramp(_am(y)), ang, W, circle, math.pi / (2 * n)), g["fbp_irad"]) < TOL_GOLD


@pytest.mark.parametrize("name", golden_names("fan_"))
def test_fanbeam_golden(name):
    g = load_golden(name)
    circle = "circle" in name
    fp = None if "default" in name else {"n_detector_pixels": 37, "detector_spacing": 0.31, "source_radius": 40.0,
                                         "detector_radius": 25.0}
    x, ang = g["x"], g["angles"]
    W = x.shape[-1]
    assert rel_err(_am(RR.fanbeam_fwd(x, ang, circle, fp)), g["y"]) < TOL_GOLD
    assert rel_err(RR.fanbeam_adj(_am(g["v"]), ang, W, circle, fp), g["At"]) < TOL_GOLD


def test_weight_sums_per_angle():
    """every per-angle weight sum of one pixel lies in [0.8, 1.35] (so below the bound of 2 the fixed-point scale assumes);
    the extremes are 1 + 4 (1 - 1/sqrt(2))^2 at 45 degrees on a lattice point and about 0.83"""
    sums = []
    for deg in np.linspace(0.0, 90.0, 91):
        th = math.radians(deg)
        for u in np.linspace(-0.5, 0.5, 11):
            for v in np.linspace(-0.5, 0.5, 11):
                sums.append(RR.pixel_weight_sums(th, u, v))
    sums = np.array(sums)
    assert sums.min() >= 0.8 and sums.max() <= 1.35 and sums.max() < 2.0, (sums.min(), sums.max())
    assert abs(RR.pixel_weight_sums(math.pi / 4, 0.0, 0.0) - (1 + 4 * (1 - 2 ** -0.5) ** 2)) < 1e-12
    assert sums.max() == pytest.approx(1 + 4 * (1 - 2 ** -0.5) ** 2, abs=1e-12)
    assert sums.min() < 0.86
