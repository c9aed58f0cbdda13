"""Pins the fp64 restatement of the 3-D blur (tests/blur3d_ref64.py) on the CPU: to the `blur3d_*` golden vectors of the real
reference (every padding, odd / even / unit filters, the four filter broadcasts, volumes smaller than the filter, the FFT
convolutions), to its own per-tap form, to adjointness, and to the exact non-finite footprint of single voxels."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import blur3d_ref64 as BR3  # noqa: E402
from conftest import golden_names, load_golden  # noqa: E402

OPERATOR_CASES = [n for n in golden_names("blur3d_") if n != "blur3d_algo"]
TOL = 1e-6  # fp32 reference against fp64, relative L2
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")  # tests/golden/make_golden_blur3d.py


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def _dot(a, b):
    return float((a.double() * b.double()).sum())


# The reference's transpose fold slices `-0:` on an axis with h // 2 == 0 (extent 1) or h // 2 - (h - 1) % 2 == 0 (extent 2):
#   * circular, extent 1 or 2, and reflect, extent 1: a shape error (RuntimeError), recorded in the fixture;
#   * replicate, extent 1: the whole axis is added onto its last index, so the fixture's A^T is not the transpose of its A.
# The 2-D drop-in computes the true transpose in both cases, and so does the 3-D one: there the restatement is pinned by
# adjointness with its own forward, which matches the reference's.
def _fold_defect(pad, fs):
    return (pad == "circular" and min(fs) <= 2) or (pad in ("replicate", "reflect") and min(fs) == 1)


def _adjoint_pair_ok(x, k, pad):
    D, H, W = x.shape[-3:]
    y = BR3.blur3d_fwd(x, k, pad)
    v = torch.randn(y.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    at = BR3.blur3d_adj(v, k, pad, D, H, W)
    return abs(_dot(y, v) - _dot(x, at)) <= 1e-10 * float(y.norm() * v.norm())


@pytest.mark.parametrize("name", OPERATOR_CASES)
def test_golden(name):
    g = load_golden(name)
    x, k = g["x"], g["k"]
    D, H, W = x.shape[-3:]
    d, h, w = fs = tuple(k.shape[-3:])
    checked = 0
    for pad in BR3.PADS:
        if f"err_{pad}" in g:
            assert ERRORS[int(g[f"err_{pad}"])] == "RuntimeError", (name, pad)
            if _fold_defect(pad, fs):
                assert _adjoint_pair_ok(x, k, pad)
            else:  # too small for valid / reflect: the drop-in's argument checks raise (tests/test_gpu_blur3d.py)
                assert (pad == "valid" and (D < d or H < h or W < w)) or (pad == "reflect" and (d // 2 >= D or h // 2 >= H or w // 2 >= W))
            continue
        a = BR3.blur3d_fwd(x, k, pad)
        assert rel(a, g[f"A_{pad}"]) < TOL, (name, pad, rel(a, g[f"A_{pad}"]))
        at = BR3.blur3d_adj(g[f"v_{pad}"], k, pad, D, H, W)
        lhs, rhs = _dot(g[f"A_{pad}"], g[f"v_{pad}"]), _dot(x, g[f"At_{pad}"])
        if _fold_defect(pad, fs):
            assert abs(lhs - rhs) > 1e-3 * (abs(lhs) + 1) and _adjoint_pair_ok(x, k, pad), (name, pad)
            continue
        assert rel(at, g[f"At_{pad}"]) < TOL, (name, pad, rel(at, g[f"At_{pad}"]))
        assert abs(lhs - rhs) <= 1e-5 * (abs(lhs) + 1), (name, pad, lhs, rhs)  # adjointness of the reference's own arrays
        checked += 1
    assert checked >= 2


@pytest.mark.parametrize("pad", BR3.PADS)
@pytest.mark.parametrize("fs", [(3, 3, 3), (4, 5, 2), (2, 1, 3), (1, 4, 4)])
def test_per_tap_form_and_adjointness(pad, fs):
    gen = torch.Generator().manual_seed(sum(fs) + len(pad))
    x = torch.randn(2, 2, 6, 7, 5, dtype=torch.float64, generator=gen)
    k = torch.randn(2, 1, *fs, dtype=torch.float64, generator=gen)
    D, H, W = x.shape[-3:]
    y = BR3.blur3d_fwd(x, k, pad)
    assert torch.allclose(y, BR3.blur3d_fwd(x, k, pad, slow=True), rtol=1e-12, atol=1e-12)
    v = torch.randn(y.shape, dtype=torch.float64, generator=gen)
    at = BR3.blur3d_adj(v, k, pad, D, H, W)
    assert torch.allclose(at, BR3.blur3d_adj(v, k, pad, D, H, W, slow=True), rtol=1e-12, atol=1e-12)
    assert abs(_dot(y, v) - _dot(x, at)) <= 1e-10 * float(y.norm() * v.norm())


def _reach(s, n, f, pad):
    """outputs (one axis) of the forward whose taps read index s"""
    if pad == "valid":
        return {i for i in range(n - f + 1) if i <= s <= i + f - 1}
    return {i for i in range(n) if any(BR3.map_index(i - u + f // 2, n, pad) == s for u in range(f))}


@pytest.mark.parametrize("pad", BR3.PADS)
@pytest.mark.parametrize("val", [float("nan"), float("inf"), float("-inf")])
def test_nonfinite_footprint(pad, val):
    """a single non-finite voxel (a corner and an interior one) reaches exactly the product of the per-axis footprints"""
    D, H, W, fs = 5, 6, 7, (3, 2, 4)
    k = torch.rand(1, 1, *fs, dtype=torch.float64, generator=torch.Generator().manual_seed(3)) + 0.1
    for loc in ((0, 0, 0), (2, 3, 5)):
        x = torch.rand(1, 1, D, H, W, dtype=torch.float64)
        x[(0, 0) + loc] = val
        y = BR3.blur3d_fwd(x, k, pad)
        want = torch.zeros(y.shape[-3:], dtype=torch.bool)
        zs, rs, cs = (sorted(_reach(s, n, f, pad)) for s, n, f in zip(loc, (D, H, W), fs))
        if zs and rs and cs:
            want[torch.tensor(zs)[:, None, None], torch.tensor(rs)[None, :, None], torch.tensor(cs)[None, None, :]] = True
        assert torch.equal(~torch.isfinite(y[0, 0]), want), (pad, loc)
        if val == val:  # an Inf keeps its sign through positive taps
            assert bool((y[0, 0][want] == val).all())
