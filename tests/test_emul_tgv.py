"""The TGV kernels (deepinv_b200/csrc/tv.cu) run on the host through the emulation, against the torch oracle
(tests/tgv_oracle.py).

The prox is driven by the package's own host side (`ops._cp_prox`, `ops.tv_drive`).  Covered: tiles at every border with H
and W not multiples of the tile edge and B*C > 1, n_it_max not a multiple of the iterations per launch K, warm restart, the break
test passing at sub-iterations 0, K - 2 and K - 1 of a launch (the replay must be bitwise the run stopped at that
iteration), ths = 0, the epsilon stencils and their adjointness, and two builds with a different tile edge and K giving
the same bits.
"""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tgv_oracle as O  # noqa: E402
from emul_tv_util import _p, image, lib, rel  # noqa: E402

from deepinv_b200 import ops  # noqa: E402

ALT = (20, 3)  # a second build: another tile edge and K, R = 32


def block(tk=None):
    t, k = C.c_int(0), C.c_int(0)
    lib(tgv=tk).dinvk_tgv_block(C.byref(t), C.byref(k))
    return t.value, k.value


def constants(lam, B, tau=0.01):
    lam = torch.as_tensor(lam, dtype=torch.float32).expand(B).contiguous()
    return (tau * (lam * 0.1)).contiguous(), (lam * 0.15).contiguous()


def prox_emul(y, lam, n_it_max=12, crit=0.0, x2=None, r2=None, u2=None, rho=1.99, check_every=2, tk=None):
    L = lib(tgv=tk)
    B, Cc, H, W = y.shape
    y = y.float().contiguous()
    tl1, l2 = constants(lam, B)
    state = [y if x2 is None else x2, torch.zeros(B, Cc, H, W, 2) if r2 is None else r2,
             torch.zeros(B, Cc, H, W, 4) if u2 is None else u2]
    (x, r, u), ctrl = ops._cp_prox(
        L, None,
        lambda xa, ra, ua, xb, rb, ub, *run: L.dinvk_tgv_prox(_p(y), xa, ra, ua, xb, rb, ub, _p(tl1), _p(l2), B, Cc, H, W, n_it_max,
                                                              crit, 0.01, rho, *run),
        state, L.dinvk_tgv_prox_workspace_bytes(B, Cc, H, W), block(tk)[1], n_it_max, check_every, fill=float("nan"))
    return x, r, u, ctrl


def test_block_constants():
    T, K = block()
    assert T >= 16 and 2 <= K <= 16
    assert block(ALT) == ALT


def test_prox_all_borders_against_oracle():
    T, K = block()
    H, W = 2 * T + 5, T + 7  # 3 x 2 tiles, partial at the bottom and right
    y = image(2, 2, H, W)
    lam = torch.tensor([0.1, 0.3])
    n = 2 * K + 3  # not a multiple of K
    x, r, u, ctrl = prox_emul(y, lam, n_it_max=n)
    xr, rr, ur, nr, _ = O.tgv_denoise(y, lam, n_it_max=n, crit=0.0)
    assert ctrl["it_done"] == nr == n
    assert ctrl["launches"] == -(-n // K)
    assert rel(x, xr) < 1e-6, rel(x, xr)
    assert rel(r, rr) < 1e-5 and rel(u, ur) < 1e-5, (rel(r, rr), rel(u, ur))


def test_warm_restart_against_oracle():
    T, K = block()
    y = image(1, 3, T + 3, T + 9, seed=1)
    x1, r1, u1, _ = prox_emul(y, 0.2, n_it_max=K + 1)
    y2 = image(1, 3, T + 3, T + 9, seed=2)
    x, r, u, _ = prox_emul(y2, 0.2, n_it_max=K, x2=x1, r2=r1, u2=u1)
    xr1, rr1, ur1, _, _ = O.tgv_denoise(y, 0.2, n_it_max=K + 1, crit=0.0)
    xr, rr, ur, _, _ = O.tgv_denoise(y2, 0.2, n_it_max=K, crit=0.0, x2=xr1, r2=rr1, u2=ur1)
    assert rel(x, xr) < 1e-6 and rel(r, rr) < 1e-5 and rel(u, ur) < 1e-5


def _crit_breaking_at(rels, target_mod, K, lo):
    """a crit whose first passing iteration index i >= lo has i % K == target_mod, with a margin of at least 1 % to the
    rel_err of iteration i and to every earlier one counted by the test (it >= 2)"""
    for i in range(max(lo, 2), len(rels)):
        if i % K != target_mod:
            continue
        prev = min(rels[2:i], default=float("inf"))
        if rels[i] < 0.99 * prev:
            return i, (rels[i] * prev) ** 0.5
    raise AssertionError("no suitable break iteration")


@pytest.mark.parametrize("where", ["first", "second_last", "last"])
def test_break_inside_a_launch_is_replayed_bitwise(where):
    T, K = block()
    y = image(2, 1, T + 9, T - 5, seed=3)
    # from x2 = 0 without over-relaxation rel_err falls steadily, so a crit between two iterations picks one of them
    kw = dict(x2=torch.zeros_like(y), rho=1.0)
    rels = []
    O.tgv_denoise(y, 0.15, n_it_max=8 * K, crit=0.0, rels=rels, **kw)
    mod = {"first": 0, "second_last": K - 2, "last": K - 1}[where]
    i, crit = _crit_breaking_at(rels, mod, K, lo=K)
    x, r, u, ctrl = prox_emul(y, 0.15, n_it_max=8 * K, crit=crit, check_every=3, **kw)
    xr, _, _, nr, _ = O.tgv_denoise(y, 0.15, n_it_max=8 * K, crit=crit, **kw)
    assert nr == i + 1 and ctrl["it_done"] == i + 1
    assert ctrl["conv_j1"] == mod + 1
    assert rel(x, xr) < 1e-6
    # the same input stopped at the break iteration by n_it_max: bitwise equal (the replay recomputes, it does not rewind)
    x0, r0, u0, _ = prox_emul(y, 0.15, n_it_max=i + 1, crit=0.0, **kw)
    assert torch.equal(x, x0) and torch.equal(r, r0) and torch.equal(u, u0)


def test_break_needs_three_iterations_and_counts_from_zero_each_call():
    y = image(1, 1, 20, 17, seed=4)
    x, r, u, ctrl = prox_emul(y, 0.1, n_it_max=40, crit=1e30)  # passes at the first allowed iteration, it = 2
    assert ctrl["it_done"] == 3 and ctrl["conv_j1"] == 2 % block()[1] + 1
    _, _, _, ctrl2 = prox_emul(y, 0.1, n_it_max=40, crit=1e30, x2=x, r2=r, u2=u)
    assert ctrl2["it_done"] == 3


def test_ths_zero_makes_everything_nan():
    y = image(1, 2, 23, 19, seed=5)
    x, r, u, _ = prox_emul(y, 0.0, n_it_max=5)
    xr, _, _, _, _ = O.tgv_denoise(y, 0.0, n_it_max=5, crit=0.0)
    assert torch.isnan(xr).all() and torch.isnan(x).all() and torch.isnan(r).all() and torch.isnan(u).all()


def test_n_it_max_zero_issues_nothing():
    y = image(1, 1, 9, 9)
    x, r, u, ctrl = prox_emul(y, 0.1, n_it_max=0)
    assert ctrl["launches"] == 0 and torch.equal(x, y) and not r.any() and not u.any()


def test_tile_and_block_change_no_bit():
    y = image(2, 2, 71, 45, seed=6)
    lam = torch.tensor([0.1, 0.4])
    a = prox_emul(y, lam, n_it_max=11)
    b = prox_emul(y, lam, n_it_max=11, tk=ALT)
    assert all(torch.equal(s, t) for s, t in zip(a[:3], b[:3]))
    kw = dict(x2=torch.zeros_like(y), rho=1.0)
    rels = []
    O.tgv_denoise(y, lam, n_it_max=30, crit=0.0, rels=rels, **kw)
    i, crit = _crit_breaking_at(rels, 1, 3, lo=5)  # inside a launch for K = 3; the default build breaks wherever i lands
    a = prox_emul(y, lam, n_it_max=30, crit=crit, **kw)
    b = prox_emul(y, lam, n_it_max=30, crit=crit, tk=ALT, **kw)
    assert a[3]["it_done"] == b[3]["it_done"] == i + 1
    assert all(torch.equal(s, t) for s, t in zip(a[:3], b[:3]))


def _stencil(op, x, out_shape, tk=None):
    out = torch.empty(out_shape)
    B, Cc, H, W = x.shape[:-1]
    assert lib(tgv=tk).dinvk_tv_stencil(op, _p(x.contiguous()), _p(out), B, Cc, H, W, None) == 0
    return out


@pytest.mark.parametrize("shape", [(2, 3, 17, 11), (1, 1, 1, 5), (1, 2, 6, 1)])
def test_epsilon_stencils_against_oracle(shape):
    g = torch.Generator().manual_seed(7)
    f = torch.randn((*shape, 2), generator=g)
    gf = torch.randn((*shape, 4), generator=g)
    assert torch.equal(_stencil(3, f, (*shape, 4)), O.tgv_epsilon(f))
    assert torch.equal(_stencil(4, gf, (*shape, 2)), O.tgv_epsilon_adjoint(gf))
    # adjointness <eps f, g> = <f, eps^T g>
    lhs = (O.tgv_epsilon(f.double()) * gf.double()).sum()
    rhs = (f.double() * _stencil(4, gf, (*shape, 2)).double()).sum()
    assert abs(float(lhs - rhs)) < 1e-5 * max(1.0, abs(float(lhs)))


def test_stencil_rejects_unknown_op():
    x = torch.zeros(1, 1, 4, 4, 4)
    assert lib().dinvk_tv_stencil(5, _p(x), _p(x), 1, 1, 4, 4, None) == 1
