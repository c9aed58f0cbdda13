"""Pin the fp64 restatement of the direct blur (tests/blur_ref64.py) on the oracle (oracle/ref_ops.py) evaluated in float64, on the
reference's own vectors (tests/golden/blur_*), on its per-tap form, on adjointness, and on the non-finite footprint it must give a
single NaN / +Inf / -Inf pixel.  CPU only."""
import itertools

import pytest
import torch

import blur_ref64 as BR
from conftest import golden_names, load_golden, rel_err
from oracle import ref_ops as R

TOL64 = 1e-12    # two fp64 evaluations of the same sums
TOL_GOLD = 1e-6  # the reference's fp32 results (the oracle in float64 agrees with them to 8.3e-8)

# (H, W, h, w): odd and even filters, h != w, filters larger than the image (single circular wrap, constant, replicate), reflect
# at its limit h//2 = H - 1, valid with a 1 x 1 output
SHAPES = [(9, 11, 3, 4), (12, 7, 5, 2), (8, 8, 4, 6), (5, 6, 7, 9), (3, 4, 5, 7), (1, 1, 1, 3), (1, 5, 2, 3), (6, 1, 4, 1),
          (4, 5, 7, 9), (7, 7, 7, 7)]


def _allowed(pad, H, W, h, w):
    if pad == "valid":
        return H >= h and W >= w
    if pad == "reflect":
        return h // 2 < H and w // 2 < W
    if pad == "circular":  # F.pad's circular mode wraps once at most
        return h // 2 <= H and w // 2 <= W and h - 1 - h // 2 <= H and w - 1 - w // 2 <= W
    return True


CASES = [(pad, *s) for pad in BR.PADS for s in SHAPES if _allowed(pad, *s)]


@pytest.mark.parametrize("pad,H,W,h,w", CASES)
@pytest.mark.parametrize("bcast", [(1, 1), (2, 1), (1, 3), (2, 3)], ids=["f11", "fB1", "f1C", "fBC"])
def test_vs_oracle64(pad, H, W, h, w, bcast):
    g = torch.Generator().manual_seed(H * 1000 + W * 100 + h * 10 + w)
    x = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64)
    k = torch.randn(*bcast, h, w, generator=g, dtype=torch.float64)
    y = BR.blur_fwd(x, k, pad)
    yr = R.blur_A(x, k, pad)
    assert y.shape == yr.shape and rel_err(y, yr) < TOL64
    v = torch.randn(*y.shape, generator=g, dtype=torch.float64)
    assert rel_err(BR.blur_adj(v, k, pad, H, W), R.blur_At(v, k, pad, H, W)) < TOL64


@pytest.mark.parametrize("pad,H,W,h,w", CASES)
def test_strips_equal_per_tap_sum(pad, H, W, h, w, monkeypatch):
    """the conv2d form (forced into one-row strips) against the plain per-tap slice sum, finite and non-finite"""
    monkeypatch.setattr(BR, "STRIP_ELEMS", 1)
    g = torch.Generator().manual_seed(7 + H + 3 * W)
    x = torch.randn(2, 1, H, W, generator=g, dtype=torch.float64)
    x[0, 0, H // 2, W // 2] = float("nan")
    x[1, 0, 0, W - 1] = float("inf")
    k = torch.randn(1, 1, h, w, generator=g, dtype=torch.float64)
    for call in ("A", "At"):
        inp = x if call == "A" else torch.randn(*BR.blur_fwd(x, k, pad).shape, generator=g, dtype=torch.float64)
        if call == "At":
            inp[0, 0, 0, 0] = float("-inf")
            inp[1, 0, -1, -1] = float("nan")
        a, b = BR.apply(call, inp, k, pad, H, W), BR.apply(call, inp, k, pad, H, W, slow=True)
        fin = torch.isfinite(b)
        assert torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a == float("inf"), b == float("inf"))
        assert torch.equal(fin, torch.isfinite(a)) and rel_err(a[fin], b[fin]) < TOL64


@pytest.mark.parametrize("name", [n for n in golden_names("blur_") if "prox" not in n])
def test_golden(name):
    g = load_golden(name)
    pad = name.split("_")[-1]
    H, W = g["x"].shape[-2:]
    assert rel_err(BR.blur_fwd(g["x"], g["filt"], pad), g["y"]) < TOL_GOLD
    assert rel_err(BR.blur_adj(g["v"], g["filt"], pad, H, W), g["At"]) < TOL_GOLD


@pytest.mark.parametrize("pad", BR.PADS)
def test_adjoint_identity64(pad):
    g = torch.Generator().manual_seed(len(pad))
    for H, W, h, w in ((13, 17, 5, 6), (9, 8, 4, 3), (6, 7, 9, 11)):
        if not _allowed(pad, H, W, h, w):
            continue
        x = torch.randn(2, 2, H, W, generator=g, dtype=torch.float64)
        k = torch.randn(2, 2, h, w, generator=g, dtype=torch.float64)
        y = BR.blur_fwd(x, k, pad)
        v = torch.randn(*y.shape, generator=g, dtype=torch.float64)
        lhs, rhs = float((y * v).sum()), float((x * BR.blur_adj(v, k, pad, H, W)).sum())
        assert abs(lhs - rhs) <= 1e-13 * abs(lhs)


def _pixels(H, W):
    """every corner and border midpoint, and the centre"""
    return sorted({(p, q) for p in (0, H // 2, H - 1) for q in (0, W // 2, W - 1)})


@pytest.mark.parametrize("pad,H,W,h,w", [c for c in CASES if c[1] * c[2] > 1] + [("replicate", 10, 12, 4, 5),
                                                                                 ("reflect", 10, 12, 5, 4)])
@pytest.mark.parametrize("call", ["A", "At"])
def test_nonfinite_footprint(pad, H, W, h, w, call):
    """one NaN / +Inf / -Inf pixel is non-finite at exactly footprint(...): the pixels that circular, replicate and reflect padding
    duplicate and the fold's corners included.  Positive filter taps: every tap that reads the pixel adds an Inf of one sign"""
    g = torch.Generator().manual_seed(H + 5 * W + 11 * h + 17 * w)
    k = torch.rand(1, 1, h, w, generator=g, dtype=torch.float64) + 0.1
    shape = (1, 1, H, W) if call == "A" else tuple(BR.blur_fwd(torch.zeros(1, 1, H, W), k, pad).shape)
    for (p, q), bad in itertools.product(_pixels(*shape[-2:]), (float("nan"), float("inf"), float("-inf"))):
        inp = torch.randn(*shape, generator=g, dtype=torch.float64)
        inp[0, 0, p, q] = bad
        out = BR.apply(call, inp, k, pad, H, W)[0, 0]
        fp = BR.footprint(call, pad, H, W, h, w, p, q)
        assert torch.equal(~torch.isfinite(out), fp), (p, q, bad)
        want = torch.isnan(out) if bad != bad else (out == bad)
        assert torch.equal(want, fp), (p, q, bad)


def test_opposite_infinities_give_nan():
    """+Inf and -Inf whose footprints overlap: NaN on the overlap, each sign on the rest of its own footprint"""
    H, W, h, w = 12, 14, 3, 5
    x = torch.zeros(1, 1, H, W, dtype=torch.float64)
    x[0, 0, 5, 6], x[0, 0, 6, 8] = float("inf"), float("-inf")
    k = torch.rand(1, 1, h, w, dtype=torch.float64) + 0.1
    for pad in BR.PADS:
        y = BR.blur_fwd(x, k, pad)[0, 0]
        fp, fm = BR.footprint("A", pad, H, W, h, w, 5, 6), BR.footprint("A", pad, H, W, h, w, 6, 8)
        assert (fp & fm).any()
        assert torch.equal(torch.isnan(y), fp & fm)
        assert torch.equal(y == float("inf"), fp & ~fm) and torch.equal(y == float("-inf"), fm & ~fp)
