"""The TV kernels (deepinv_b200/csrc/tv.cu) run on the host through the emulation, against the torch oracle (tests/tv_oracle.py).

The prox is driven by the package's own host side (`ops._cp_prox`, `ops.tv_drive`).  Covered: tiles at every border with H
and W not multiples of the tile edge and B*C > 1, n_it_max not a multiple of the iterations per launch K, the break test
passing at sub-iterations 0, K - 2 and K - 1 of a launch (the replay must be bitwise the run stopped at that iteration),
warm restart, both dual projections, the stencils, and two builds with a different tile edge and K giving the same bits.
"""
import ctypes as C
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import tv_oracle as O  # noqa: E402
from emul_tv_util import _p, image, lib, rel  # noqa: E402

from deepinv_b200 import ops  # noqa: E402

ALT = (20, 3)  # a second build: another tile edge and K, R = 26


def prox_emul(y, lam, l1=False, n_it_max=20, crit=0.0, x2=None, u2=None, tau=0.01, rho=1.99, check_every=2, tk=None):
    L = lib(tv=tk)
    B, Cc, H, W = y.shape
    y = y.float().contiguous()
    lam = torch.as_tensor(lam, dtype=torch.float32).expand(B).contiguous()
    state = [y if x2 is None else x2, torch.zeros(B, Cc, H, W, 2) if u2 is None else u2]
    (x, u), ctrl = ops._cp_prox(
        L, None,
        lambda xa, ua, xb, ub, *run: L.dinvk_tv_prox(_p(y), xa, ua, xb, ub, _p(lam), B, Cc, H, W, n_it_max, crit, tau, rho, int(l1),
                                                     *run),
        state, L.dinvk_tv_prox_workspace_bytes(B, Cc, H, W), block(tk)[1], n_it_max, check_every, fill=float("nan"))
    return x, u, ctrl


def block(tk=None):
    t, k = C.c_int(0), C.c_int(0)
    lib(tv=tk).dinvk_tv_block(C.byref(t), C.byref(k))
    return t.value, k.value


def test_block_constants():
    T, K = block()
    assert T >= 16 and 2 <= K <= 16
    assert block(ALT) == ALT


@pytest.mark.parametrize("l1", [False, True])
def test_prox_all_borders_against_oracle(l1):
    T, K = block()
    H, W = 2 * T + 5, T + 7  # 3 x 2 tiles, partial at the bottom and right
    y = image(2, 2, H, W)
    lam = torch.tensor([0.1, 0.25])
    n = 2 * K + 3  # not a multiple of K
    x, u, ctrl = prox_emul(y, lam, l1=l1, n_it_max=n)
    xr, ur, nr, _ = O.tv_denoise(y, lam, l1=l1, n_it_max=n, crit=0.0)
    assert ctrl["it_done"] == nr == n
    assert ctrl["launches"] == -(-n // K)
    assert rel(x, xr) < 1e-6, rel(x, xr)
    assert rel(u, ur) < 1e-5, rel(u, ur)


def test_warm_restart_against_oracle():
    T, K = block()
    y = image(1, 3, T + 3, 2 * T + 1, seed=1)
    x1, u1, _ = prox_emul(y, 0.2, n_it_max=K + 1)
    y2 = image(1, 3, T + 3, 2 * T + 1, seed=2)
    x, u, ctrl = prox_emul(y2, 0.2, n_it_max=K, x2=x1, u2=u1)
    xr1, ur1, _, _ = O.tv_denoise(y, 0.2, n_it_max=K + 1, crit=0.0)
    xr, ur, _, _ = O.tv_denoise(y2, 0.2, n_it_max=K, crit=0.0, x2=xr1, u2=ur1)
    assert rel(x, xr) < 1e-6 and rel(u, ur) < 1e-5


def _crit_breaking_at(rels, target_mod, K, lo=2):
    """a crit whose first passing iteration index i >= lo has i % K == target_mod, with a margin of at least 0.25 % to the
    rel_err of iteration i and to every earlier one"""
    for i in range(max(lo, 2), len(rels)):
        if i % K != target_mod:
            continue
        prev = min(rels[2:i], default=float("inf"))
        if rels[i] < 0.995 * prev:
            return i, (rels[i] * prev) ** 0.5
    raise AssertionError("no suitable break iteration")


@pytest.mark.parametrize("where", ["first", "second_last", "last"])
def test_break_inside_a_launch_is_replayed_bitwise(where):
    T, K = block()
    y = image(2, 1, T + 9, T - 5, seed=3)
    rels = []
    rho = 1.0  # without over-relaxation rel_err decreases steadily, so a crit between two iterations picks one of them
    O.tv_denoise(y, 0.15, rho=rho, n_it_max=6 * K, crit=0.0, rels=rels)
    mod = {"first": 0, "second_last": K - 2, "last": K - 1}[where]
    i, crit = _crit_breaking_at(rels, mod, K, lo=K)
    x, u, ctrl = prox_emul(y, 0.15, rho=rho, n_it_max=6 * K, crit=crit, check_every=3)
    xr, ur, nr, _ = O.tv_denoise(y, 0.15, rho=rho, n_it_max=6 * K, crit=crit)
    assert nr == i + 1 and ctrl["it_done"] == i + 1
    assert ctrl["conv_j1"] == mod + 1
    assert rel(x, xr) < 1e-6
    # the same input stopped at the break iteration by n_it_max: bitwise equal (the replay recomputes, it does not rewind)
    x0, u0, c0 = prox_emul(y, 0.15, rho=rho, n_it_max=i + 1, crit=0.0)
    assert torch.equal(x, x0) and torch.equal(u, u0)


def test_break_needs_three_iterations_and_counts_from_zero_each_call():
    y = image(1, 1, 20, 17, seed=4)
    x, u, ctrl = prox_emul(y, 0.1, n_it_max=40, crit=1e30)  # passes at the first allowed iteration, it = 2
    assert ctrl["it_done"] == 3
    x2, u2, ctrl2 = prox_emul(y, 0.1, n_it_max=40, crit=1e30, x2=x, u2=u)
    assert ctrl2["it_done"] == 3


def test_ths_zero_keeps_the_image_and_nan_only_where_unread():
    y = image(1, 2, 23, 19, seed=5)  # noisy: no flat regions
    x, u, _ = prox_emul(y, 0.0, n_it_max=12)
    xr, ur, _, _ = O.tv_denoise(y, 0.0, n_it_max=12, crit=0.0)
    assert torch.equal(torch.isnan(x), torch.isnan(xr)) and not torch.isnan(x).any()
    assert rel(x, xr) < 1e-6 and rel(x, y) < 1e-6
    read0, read1 = u[:, :, :-1, :, 0], u[:, :, :, :-1, 1]  # the components nabla_adjoint reads
    assert torch.equal(read0, ur[:, :, :-1, :, 0]) and torch.equal(read1, ur[:, :, :, :-1, 1])


def test_n_it_max_zero_issues_nothing():
    y = image(1, 1, 9, 9)
    x, u, ctrl = prox_emul(y, 0.1, n_it_max=0)
    assert ctrl["launches"] == 0 and torch.equal(x, y) and not u.any()


def test_tile_and_block_change_no_bit():
    y = image(2, 2, 71, 45, seed=6)
    lam = torch.tensor([0.1, 0.4])
    for l1 in (False, True):
        a = prox_emul(y, lam, l1=l1, n_it_max=11)
        b = prox_emul(y, lam, l1=l1, n_it_max=11, tk=ALT)
        assert all(torch.equal(s, t) for s, t in zip(a[:2], b[:2]))
    rels = []
    O.tv_denoise(y, lam, rho=1.0, n_it_max=30, crit=0.0, rels=rels)
    i, crit = _crit_breaking_at(rels, 1, 3, lo=5)  # inside a launch for K = 3; the default build breaks wherever i lands
    a = prox_emul(y, lam, rho=1.0, n_it_max=30, crit=crit)
    b = prox_emul(y, lam, rho=1.0, n_it_max=30, crit=crit, tk=ALT)
    assert a[2]["it_done"] == b[2]["it_done"] == i + 1
    assert all(torch.equal(s, t) for s, t in zip(a[:2], b[:2]))


def _stencil(op, x, out_shape):
    out = torch.empty(out_shape)
    B, Cc, H, W = (x.shape if op != 1 else x.shape[:-1])
    assert lib().dinvk_tv_stencil(op, _p(x.contiguous()), _p(out), B, Cc, H, W, None) == 0
    return out


@pytest.mark.parametrize("shape", [(2, 3, 17, 11), (1, 1, 1, 5), (1, 2, 6, 1)])
def test_stencils_and_fn_against_oracle(shape):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(shape, generator=g)
    x[..., : shape[2] // 2, : shape[3] // 2] = 0.5  # a flat patch: |Dx| = 0 there
    gr = torch.randn((*shape, 2), generator=g)
    assert torch.equal(_stencil(0, x, (*shape, 2)), O.tv_nabla(x))
    assert torch.equal(_stencil(1, gr, shape), O.tv_nabla_adjoint(gr))
    assert rel(_stencil(2, x, shape), O.tv_grad(x)) < 1e-6 if O.tv_grad(x).norm() > 0 else True
    # adjointness <D x, g> = <x, D^T g> (the reference's test_models check)
    lhs = (O.tv_nabla(x.double()) * gr.double()).sum()
    rhs = (x.double() * _stencil(1, gr, shape).double()).sum()
    assert abs(float(lhs - rhs)) < 1e-5 * max(1.0, abs(float(lhs)))
    for l1 in (False, True):
        B = shape[0]
        nb = lib().dinvk_tv_fn_workspace_bytes(*shape)
        ws = torch.zeros(nb // 8 + 1, dtype=torch.float64)
        out = torch.empty(B)
        assert lib().dinvk_tv_fn(_p(out), _p(x), int(l1), *shape, _p(ws), nb, None) == 0
        ref = O.tv_fn(x.double(), l1=l1).float()
        assert torch.allclose(out, ref, rtol=1e-6, atol=1e-6)
