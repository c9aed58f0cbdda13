"""MATLAB-bicubic resize (deepinv/physics/functional/imresize.py) on libdinvk's fused resize kernels.

`imresize_matlab` applies resize_1d (:222-296) to H then W.  Per axis the resize is a banded matrix M (n_out x n_in); its
tables are built here once per (n_in, n_out, scale, antialiasing) with the reference's own torch arithmetic on the CPU in
fp32, so the weights are the reference's bits, and kept on the device:
  - forward  : `base` (n_out,) int32, the unreflected first tap of each output, and `weight` (n_out, k) fp32;
  - transpose: CSR by input index (`ptr`, `out`, `wt`), every (output, tap) pair that lands on an input, reflection folds
    included, sorted by output index.
`dinvk_resize_fwd` applies both passes in one launch, `dinvk_resize_adj` the exact transpose in one launch.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
from torch import Tensor

from .. import ops
from .forward import linear_apply


def _cubic_contribution(x: Tensor, a: float = -0.5) -> Tensor:
    """imresize.py:23-38, op for op"""
    ax = x.abs()
    ax2 = ax * ax
    ax3 = ax * ax2
    range_01 = ax.le(1)
    range_12 = torch.logical_and(ax.gt(1), ax.le(2))
    cont_01 = (a + 2) * ax3 - (a + 3) * ax2 + 1
    cont_01 = cont_01 * range_01.to(dtype=x.dtype)
    cont_12 = (a * ax3) - (5 * a * ax2) + (8 * a * ax) - (4 * a)
    cont_12 = cont_12 * range_12.to(dtype=x.dtype)
    return cont_01 + cont_12


@dataclass
class AxisTable:
    """one axis of the resize, host copies (built once) and a per-device cache of the uploaded tensors"""

    n_in: int
    n_out: int
    scale: float
    k: int
    base: Tensor    # (n_out,) int32
    weight: Tensor  # (n_out, k) fp32
    ptr: Tensor     # (n_in + 1,) int32
    out: Tensor     # (nnz,) int32
    wt: Tensor      # (nnz,) fp32

    def __post_init__(self):
        self._dev = {}

    def on(self, dev: torch.device) -> tuple[Tensor, ...]:
        key = str(dev)
        if key not in self._dev:
            self._dev[key] = tuple(t.to(dev) for t in (self.base, self.weight, self.ptr, self.out, self.wt))
        return self._dev[key]


_TABLES: dict[tuple, AxisTable] = {}


def axis_table(n_in: int, size: int, scale: float, antialiasing: bool = True) -> AxisTable:
    """the cubic resize_1d of an n_in-sample axis to `size` samples at `scale` (imresize.py:222-296, kernel 'cubic', reflect
    padding), as tables.  Raises the IndexError the reference's reflect_padding raises when the band reaches more than n_in
    samples past an edge."""
    key = (n_in, size, float(scale), bool(antialiasing))
    tab = _TABLES.get(key)
    if tab is not None:
        return tab
    kernel_size = 4
    if antialiasing and scale < 1:
        antialiasing_factor = scale
        kernel_size = math.ceil(kernel_size / antialiasing_factor)
    else:
        antialiasing_factor = 1
    kernel_size += 2
    pos = torch.linspace(0, size - 1, steps=size, dtype=torch.float32)
    pos = (pos + 0.5) / scale - 0.5
    base = pos.floor() - (kernel_size // 2) + 1
    dist = pos - base
    buffer_pos = dist.new_zeros(kernel_size, len(dist))
    for idx, buffer_sub in enumerate(buffer_pos):
        buffer_sub.copy_(dist - idx)
    buffer_pos *= antialiasing_factor
    weight = _cubic_contribution(buffer_pos)
    weight /= weight.sum(dim=0, keepdim=True)
    base = base.long()
    pad_pre = max(0, -int(base.min()))
    pad_post = max(0, int(base.max()) + kernel_size - 1 - n_in + 1)
    # reflect_padding copies x[p] for p < pad_pre and x[-(p + 1)] for p < pad_post: the first index past the axis fails
    if pad_pre > n_in:
        raise IndexError(f"index {n_in} is out of bounds for dimension 1 with size {n_in}")
    if pad_post > n_in:
        raise IndexError(f"index {-(n_in + 1)} is out of bounds for dimension 1 with size {n_in}")
    # transpose: the reflected input of every (output, tap), sorted by (input, output, tap)
    j = base[:, None] + torch.arange(kernel_size)[None, :]
    j = torch.where(j < 0, -1 - j, torch.where(j >= n_in, 2 * n_in - 1 - j, j))
    o = torch.arange(size)[:, None].expand_as(j)
    wt = weight.t().contiguous()
    order = torch.argsort(j.reshape(-1) * (size * kernel_size) + torch.arange(size * kernel_size), stable=True)
    ptr = torch.zeros(n_in + 1, dtype=torch.int64)
    ptr[1:] = torch.cumsum(torch.bincount(j.reshape(-1), minlength=n_in), 0)
    tab = AxisTable(n_in, size, float(scale), kernel_size, base.to(torch.int32), wt, ptr.to(torch.int32),
                    o.reshape(-1)[order].to(torch.int32).contiguous(), wt.reshape(-1)[order].contiguous())
    _TABLES[key] = tab
    return tab


def _resize_fwd(x: Tensor, th: AxisTable | None, tw: AxisTable | None) -> Tensor:
    """(B, C, H, W) -> (B, C, Ho, Wo); an axis with table None is the identity (scale 1)"""
    B, C, H, W = x.shape
    th = th or _identity(H)
    tw = tw or _identity(W)
    return ops.resize_fwd(x, th, tw)


def _resize_adj(y: Tensor, th: AxisTable | None, tw: AxisTable | None, H: int, W: int) -> Tensor:
    th = th or _identity(H)
    tw = tw or _identity(W)
    return ops.resize_adj(y, th, tw)


def _identity(n: int) -> AxisTable:
    """scale 1 on one axis while the other resizes: resize_1d returns its input, here a one-tap band"""
    key = ("identity", n)
    tab = _TABLES.get(key)
    if tab is None:
        idx = torch.arange(n, dtype=torch.int32)
        one = torch.ones(n, dtype=torch.float32)
        tab = AxisTable(n, n, 1.0, 1, idx, one[:, None].contiguous(), torch.arange(n + 1, dtype=torch.int32), idx, one)
        _TABLES[key] = tab
    return tab


def resize_plan(h: int, w: int, scale=None, sizes=None, antialiasing: bool = True, kernel: str = "cubic",
                padding_type: str | None = "reflect"):
    """output size and per-axis tables (None: that axis is left as it is) of imresize_matlab on an (h, w) image.  Errors come in
    the reference's order: kernel, then padding type, then a band reaching past the image (H before W)."""
    if sizes is None:
        sizes = (math.ceil(h * scale), math.ceil(w * scale))
        scales = (scale, scale)
    if scale is None:
        scales = (sizes[0] / h, sizes[1] / w)
    if scales[0] != 1 or scales[1] != 1:
        if kernel == "gaussian":
            raise NotImplementedError("imresize_matlab: only the 'cubic' kernel runs on the library's kernels")
        if kernel != "cubic":
            raise ValueError("{} kernel is not supported!".format(kernel))
        if padding_type is None:
            raise NotImplementedError("imresize_matlab: padding_type=None is not supported; use 'reflect'")
        if padding_type != "reflect":
            raise ValueError("{} padding is not supported!".format(padding_type))
    th = None if scales[0] == 1 else axis_table(h, sizes[0], scales[0], antialiasing)
    tw = None if scales[1] == 1 else axis_table(w, sizes[1], scales[1], antialiasing)
    out = (th.n_out if th is not None else h, tw.n_out if tw is not None else w)
    return out, th, tw


def resize(x: Tensor, th: AxisTable | None, tw: AxisTable | None) -> Tensor:
    """the resize of (B, C, H, W) x, differentiable in x through the transpose kernel"""
    if th is None and tw is None:
        return x
    H, W = x.shape[-2:]
    return linear_apply(x, lambda t: _resize_fwd(t, th, tw), lambda t: _resize_adj(t, th, tw, H, W))


def resize_adjoint(y: Tensor, th: AxisTable | None, tw: AxisTable | None, H: int, W: int) -> Tensor:
    """the transpose of `resize` onto (B, C, H, W), differentiable in y through the forward kernel"""
    if th is None and tw is None:
        return y
    return linear_apply(y, lambda t: _resize_adj(t, th, tw, H, W), lambda t: _resize_fwd(t, th, tw))


def imresize_matlab(x: Tensor, scale: float | None = None, sizes: tuple[int, int] | None = None, kernel: str = "cubic",
                    sigma: float = 2, padding_type: str = "reflect", antialiasing: bool = True) -> Tensor:
    r"""MATLAB imresize (deepinv/physics/functional/imresize.py:299-372) with the bicubic kernel and reflect padding, on
    (H, W), (C, H, W) or (B, C, H, W) fp32 CUDA tensors.  `scale` > 1 upsamples.  One fused launch; differentiable in x."""
    if scale is None and sizes is None:
        raise ValueError("One of scale or sizes must be specified!")
    if scale is not None and sizes is not None:
        raise ValueError("Please specify scale or sizes to avoid conflict!")
    if x.dim() not in (2, 3, 4):
        raise ValueError("{}-dim Tensor is not supported!".format(x.dim()))
    h, w = x.shape[-2:]
    out, th, tw = resize_plan(h, w, scale, sizes, antialiasing, kernel, padding_type)
    lead = x.shape[:-2]
    x4 = x.reshape(-1, 1, h, w)
    if x4.dtype != torch.float32:
        raise NotImplementedError(f"imresize_matlab: fp32 tensors only, got {x.dtype}")
    y = resize(x4, th, tw)
    return y.reshape(*lead, *out)
