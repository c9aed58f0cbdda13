"""fp64 restatement of MATLAB-bicubic imresize (deepinv/physics/functional/imresize.py:222-372, kernel 'cubic', reflect
padding) as dense per-axis matrices: y = M_H x M_W^T on every (b, c) plane, A^T y = M_H^T y M_W.

Written from the definition, not from the library: positions pos = (i + 0.5) / scale - 0.5, k = ceil(4 / scale) + 2 taps with
antialiasing (4 + 2 without, or when upsampling) starting at floor(pos) - k // 2 + 1, cubic weights (a = -0.5) of the
distance times the antialiasing factor, normalised to sum 1; taps outside [0, n) reflect with the edge sample repeated.
`dtype=torch.float32` evaluates the same definition in fp32 throughout (positions, weights, products): an fp32 reference of
the operator, whose tap positions round as the reference's own do.
"""
from __future__ import annotations

import math

import torch


def cubic(x: torch.Tensor, a: float = -0.5) -> torch.Tensor:
    ax = x.abs()
    inner = (a + 2) * ax ** 3 - (a + 3) * ax ** 2 + 1
    outer = a * ax ** 3 - 5 * a * ax ** 2 + 8 * a * ax - 4 * a
    return torch.where(ax <= 1, inner, torch.where(ax <= 2, outer, torch.zeros_like(ax)))


def matrix(n_in: int, n_out: int, scale: float, antialiasing: bool = True, dtype=torch.float64) -> torch.Tensor:
    """M (n_out, n_in) of one axis"""
    if scale == 1:
        return torch.eye(n_in, dtype=dtype)
    aa = scale if (antialiasing and scale < 1) else 1.0
    k = (math.ceil(4 / aa) if aa != 1 else 4) + 2
    i = torch.arange(n_out, dtype=dtype)
    pos = (i + 0.5) / scale - 0.5
    base = torch.floor(pos) - k // 2 + 1
    t = torch.arange(k, dtype=dtype)
    w = cubic((pos[:, None] - base[:, None] - t[None, :]) * aa)
    w = w / w.sum(1, keepdim=True)
    j = (base[:, None] + t[None, :]).long()
    if int(j.min()) < -n_in or int(j.max()) > 2 * n_in - 1:
        raise IndexError(f"the band reaches more than {n_in} samples past the axis")
    j = torch.where(j < 0, -1 - j, torch.where(j >= n_in, 2 * n_in - 1 - j, j))
    M = torch.zeros(n_out, n_in, dtype=dtype)
    M.scatter_add_(1, j, w)
    return M


def sizes_for(h: int, w: int, scale: float) -> tuple[int, int]:
    return math.ceil(h * scale), math.ceil(w * scale)


def operators(h: int, w: int, scale: float, antialiasing: bool = True, dtype=torch.float64):
    """(M_H, M_W) of imresize_matlab(scale=...) on an (h, w) image"""
    ho, wo = sizes_for(h, w, scale)
    return matrix(h, ho, scale, antialiasing, dtype), matrix(w, wo, scale, antialiasing, dtype)


def apply(x: torch.Tensor, MH: torch.Tensor, MW: torch.Tensor) -> torch.Tensor:
    x = x.to(MH.dtype)
    return torch.matmul(torch.matmul(MH, x), MW.t())


def apply_t(y: torch.Tensor, MH: torch.Tensor, MW: torch.Tensor) -> torch.Tensor:
    y = y.to(MH.dtype)
    return torch.matmul(torch.matmul(MH.t(), y), MW)


def imresize(x: torch.Tensor, scale: float, antialiasing: bool = True) -> torch.Tensor:
    MH, MW = operators(*x.shape[-2:], scale, antialiasing)
    return apply(x, MH, MW)


def downsample_adjoint(y: torch.Tensor, factor: int, antialiasing: bool = True) -> torch.Tensor:
    """DownsamplingMatlab.A_adjoint: the transpose on the (H_out f, W_out f) image"""
    H, W = y.shape[-2] * factor, y.shape[-1] * factor
    MH, MW = operators(H, W, 1 / factor, antialiasing)
    return apply_t(y, MH, MW)
