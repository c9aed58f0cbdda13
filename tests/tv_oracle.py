"""Test oracle for total variation: deepinv/models/tv.py and deepinv/optim/prior.py:485-611 restated in plain torch.

Any dtype (fp32 to follow the reference bit for bit where torch does, fp64 as the yardstick) and any device.
`tv_denoise` also returns the iteration count and the last rel_err, which the reference computes but does not return.
"""
from __future__ import annotations

import torch


def tv_nabla(x: torch.Tensor) -> torch.Tensor:
    """(B,C,H,W) -> (B,C,H,W,2); component 0 = vertical difference (zero last row), 1 = horizontal (zero last column)"""
    u = torch.zeros((*x.shape, 2), device=x.device, dtype=x.dtype)
    u[:, :, :-1, :, 0] = x[:, :, 1:] - x[:, :, :-1]
    u[:, :, :, :-1, 1] = x[:, :, :, 1:] - x[:, :, :, :-1]
    return u


def tv_nabla_adjoint(g: torch.Tensor) -> torch.Tensor:
    """(B,C,H,W,2) -> (B,C,H,W), in the reference's order of updates"""
    u = torch.zeros(g.shape[:-1], device=g.device, dtype=g.dtype)
    u[:, :, :-1] -= g[:, :, :-1, :, 0]
    u[:, :, 1:] += g[:, :, :-1, :, 0]
    u[:, :, :, :-1] -= g[:, :, :, :-1, 1]
    u[:, :, :, 1:] += g[:, :, :, :-1, 1]
    return u


def _lambd(ths, B, dtype, device):
    if isinstance(ths, torch.Tensor):
        lam = ths.squeeze().to(dtype=dtype, device=device)
    else:
        lam = torch.tensor(float(ths), dtype=dtype, device=device)
    if lam.dim() == 0:
        lam = lam.expand(B)
    return lam.reshape(B, 1, 1, 1, 1)


def tv_denoise(y: torch.Tensor, ths, l1: bool = False, tau: float = 0.01, rho: float = 1.99, n_it_max: int = 1000,
               crit: float = 1e-5, x2: torch.Tensor | None = None, u2: torch.Tensor | None = None, rels: list | None = None):
    """TVDenoiser / TVL1Denoiser forward from (x2, u2) (None: the restart y, 0).  Returns (x2, u2, iterations, rel_err);
    `rels`, if given, receives every iteration's rel_err."""
    x2 = y.clone() if x2 is None else x2.clone()
    u2 = torch.zeros((*y.shape, 2), device=y.device, dtype=y.dtype) if u2 is None else u2.clone()
    sigma = 1 / tau / 2 ** (y.ndim - 1)
    lam = _lambd(ths, y.shape[0], y.dtype, y.device)
    it, rel = 0, float("nan")
    for it in range(n_it_max):
        x_prev = x2
        x = (x2 - tau * tv_nabla_adjoint(u2) + tau * y) / (1 + tau)
        t = u2 + sigma * tv_nabla(2 * x - x2)
        if l1:
            u = torch.clamp(t, -lam, lam)
        else:
            u = t / torch.clamp(torch.linalg.vector_norm(t, dim=-1, ord=2, keepdim=True) / lam, min=1.0)
        x2 = x2 + rho * (x - x2)
        u2 = u2 + rho * (u - u2)
        rel_t = torch.linalg.norm(x_prev.flatten() - x2.flatten()) / torch.linalg.norm(x2.flatten() + 1e-12)
        rel = float(rel_t)
        if rels is not None:
            rels.append(rel)
        if it > 1 and rel_t < crit:
            return x2, u2, it + 1, rel
    return x2, u2, (it + 1 if n_it_max > 0 else 0), rel


def tv_fn(x: torch.Tensor, l1: bool = False) -> torch.Tensor:
    g = tv_nabla(x)
    y = torch.sum(torch.abs(g), dim=-1) if l1 else torch.sqrt(torch.sum(g ** 2, dim=-1))
    return torch.sum(y.reshape(x.shape[0], -1), dim=-1)


def tv_grad(x: torch.Tensor) -> torch.Tensor:
    dx = tv_nabla(x)
    n = torch.linalg.vector_norm(dx, dim=-1, keepdim=True)
    nz = n > 0
    return tv_nabla_adjoint(torch.where(nz, dx / torch.where(nz, n, torch.ones_like(n)), torch.zeros_like(dx)))
