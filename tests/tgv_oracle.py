"""Test oracle for total generalized variation: deepinv/models/tgv.py (2-D) restated in plain torch.

Any dtype (fp32 to follow the reference bit for bit where torch does, fp64 as the yardstick) and any device.
`tgv_denoise` also returns the iteration count and the last rel_err, which the reference computes but does not return.
The sums over the last axis are written out left to right, ((a + b) + c) + d, which is how torch's CPU `sum(.., -1)`
rounds them for these short rows; a pairwise order would differ in the last bit.
"""
from __future__ import annotations

import torch

from tv_oracle import tv_nabla, tv_nabla_adjoint


def tgv_epsilon(f: torch.Tensor) -> torch.Tensor:
    """(B,C,H,W,2) -> (B,C,H,W,4): component 2i + j = backward difference of f_i along axis j (0: H, 1: W), zero first row"""
    g = torch.zeros((*f.shape[:-1], 4), device=f.device, dtype=f.dtype)
    for i in range(2):
        g[:, :, 1:, :, 2 * i] = f[:, :, 1:, :, i] - f[:, :, :-1, :, i]
        g[:, :, :, 1:, 2 * i + 1] = f[:, :, :, 1:, i] - f[:, :, :, :-1, i]
    return g


def tgv_epsilon_adjoint(g: torch.Tensor) -> torch.Tensor:
    """(B,C,H,W,4) -> (B,C,H,W,2), in the reference's order of updates"""
    f = torch.zeros((*g.shape[:-1], 2), device=g.device, dtype=g.dtype)
    for i in range(2):
        f[:, :, :-1, :, i] -= g[:, :, 1:, :, 2 * i]
        f[:, :, 1:, :, i] += g[:, :, 1:, :, 2 * i]
        f[:, :, :, :-1, i] -= g[:, :, :, 1:, 2 * i + 1]
        f[:, :, :, 1:, i] += g[:, :, :, 1:, 2 * i + 1]
    return f


def _sq_sum_last(v: torch.Tensor) -> torch.Tensor:
    """sum of squares over the last axis, left to right"""
    s = v[..., 0] * v[..., 0]
    for k in range(1, v.shape[-1]):
        s = s + v[..., k] * v[..., k]
    return s


def _lambd(ths, B, dtype, device):
    if isinstance(ths, torch.Tensor):
        lam = ths.squeeze().to(dtype=dtype, device=device)
    else:
        lam = torch.tensor(float(ths), dtype=dtype, device=device)
    if lam.dim() == 0:
        lam = lam.expand(B)
    return lam.reshape(B, 1, 1, 1)


def tgv_denoise(y: torch.Tensor, ths, n_it_max: int = 1000, crit: float = 1e-5, x2: torch.Tensor | None = None,
                r2: torch.Tensor | None = None, u2: torch.Tensor | None = None, tau: float = 0.01, rho: float = 1.99,
                rels: list | None = None):
    """TGVDenoiser forward from (x2, r2, u2) (None: the restart y, 0, 0).  Returns (x2, r2, u2, iterations, rel_err);
    `rels`, if given, receives every iteration's rel_err."""
    x2 = y.clone() if x2 is None else x2.clone()
    r2 = torch.zeros((*y.shape, 2), device=y.device, dtype=y.dtype) if r2 is None else r2.clone()
    u2 = torch.zeros((*y.shape, 4), device=y.device, dtype=y.dtype) if u2 is None else u2.clone()
    sigma = 1 / tau / 72
    lam = _lambd(ths, y.shape[0], y.dtype, y.device)
    lambda1, lambda2 = lam * 0.1, lam * 0.15
    one = torch.ones((), device=y.device, dtype=y.dtype)
    it, rel = 0, float("nan")
    for it in range(n_it_max):
        x_prev = x2
        tmp = tau * tgv_epsilon_adjoint(u2)
        x = ((x2 - tv_nabla_adjoint(tmp)) + tau * y) / (1 + tau)
        s = r2 + tmp
        m = torch.maximum(torch.sqrt(_sq_sum_last(s)) / (tau * lambda1), one).unsqueeze(-1)
        r = s - s / m
        t = u2 + sigma * tgv_epsilon(tv_nabla(2 * x - x2) - (2 * r - r2))
        u = t / torch.maximum(torch.sqrt(_sq_sum_last(t)) / lambda2, one).unsqueeze(-1)
        x2 = x2 + rho * (x - x2)
        r2 = r2 + rho * (r - r2)
        u2 = u2 + rho * (u - u2)
        rel_t = torch.linalg.norm(x_prev.flatten() - x2.flatten()) / (torch.linalg.norm(x2.flatten()) + 1e-12)
        rel = float(rel_t)
        if rels is not None:
            rels.append(rel)
        if it > 1 and rel_t < crit:
            return x2, r2, u2, it + 1, rel
    return x2, r2, u2, (it + 1 if n_it_max > 0 else 0), rel
