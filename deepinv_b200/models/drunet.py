"""DRUNet on libdinvk's convolution kernels.

Drop-in for deepinv/models/drunet.py:23-263: same constructor, same module tree (so
`state_dict()` keys and shapes are identical and the reference's weights load with
`load_state_dict`), same `forward(x, sigma)` noise-level handling (:212-249), same padding / split
rules for awkward sizes (:252-262, models/utils.py:49-101).  The nn.Conv2d / ConvTranspose2d modules
below only hold the parameters; the arithmetic is `dinvk_conv_f32` (fp32 parity path) or the
wgmma bf16 implicit GEMM (`precision="bf16"`, see deepinv_b200/models/tc_engine.py).

Layer list for the reference configuration (SURVEY Appendix A.12): head 3x3, 4 scales of 4 ResBlocks
(x + conv(relu(conv(x)))) with 2x2/s2 down-convs, 4 body ResBlocks, 2x2/s2 transposed up-convs with
additive skips, tail 3x3; every conv is bias-free.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .base import Denoiser, _no_grad_guard


_CONV = {2: (nn.Conv2d, nn.ConvTranspose2d), 3: (nn.Conv3d, nn.ConvTranspose3d)}


class ResBlock(nn.Module):
    """x + conv(relu(conv(x)))  (drunet.py:400-433); parameters live at res.0 / res.2 like the reference"""

    def __init__(self, channels: int, bias: bool = False, dim: int = 2):
        super().__init__()
        conv = _CONV[dim][0]
        self.res = nn.Sequential(
            conv(channels, channels, 3, 1, 1, bias=bias),
            nn.ReLU(inplace=True),
            conv(channels, channels, 3, 1, 1, bias=bias),
        )


def _stage(channels_in, channels_out, nb, down: bool, dim: int = 2):
    conv, convt = _CONV[dim]
    blocks = [ResBlock(channels_in, dim=dim) for _ in range(nb)]
    if down:
        return nn.Sequential(*blocks, conv(channels_in, channels_out, 2, 2, 0, bias=False))
    return nn.Sequential(convt(channels_in, channels_out, 2, 2, 0, bias=False),
                         *[ResBlock(channels_out, dim=dim) for _ in range(nb)])


def body_blocks(m) -> list:
    """the ResBlocks of m_body (a single unwrapped ResBlock when a 3-D model has nb = 1, as in the reference)"""
    return [m.m_body] if isinstance(m.m_body, ResBlock) else list(m.m_body)


def fix_dim(dim) -> int:
    """2 / 3 from an int or a string such as "3", "3d", "2D" (the reference's models/utils.py:105-125)"""
    if isinstance(dim, str):
        if len(dim) == 1:
            dim_int = int(dim)
        elif len(dim) == 2:
            dim_int = int(dim[0])
        else:
            raise ValueError(f"dim must be int, or '3', '2d', '3D', etc., got {dim}")
    elif isinstance(dim, int):
        dim_int = dim
    else:
        raise ValueError(f"dim must be of type str or int, got {dim} ({type(dim)})")
    if dim_int not in [2, 3]:
        raise ValueError(f"Only 2D or 3D architectures are supported, got dim={dim_int}")
    return dim_int


def weights_init_drunet(m):
    if m.__class__.__name__.find("Conv") != -1:
        nn.init.orthogonal_(m.weight.data, gain=0.2)


class DRUNet(Denoiser):
    def __init__(self, in_channels: int = 3, out_channels: int = 3, nc=(64, 128, 256, 512), nb: int = 4,
                 act_mode: str = "R", downsample_mode: str = "strideconv", upsample_mode: str = "convtranspose",
                 pretrained: str | None = "download", pretrained_2d_isotropic: bool = False, device=None, dim=2,
                 precision: str = "fp32"):
        super().__init__()
        dim = fix_dim(dim)
        if act_mode != "R" or downsample_mode != "strideconv" or upsample_mode != "convtranspose":
            raise NotImplementedError("deepinv_b200.DRUNet implements the reference's default architecture "
                                      "(ReLU, strided-conv down, conv-transpose up)")
        if dim == 3 and precision == "bf16":
            raise NotImplementedError("DRUNet(dim=3) runs at precision 'fp32', 'tc32' or 'tc32h'; the bf16 engine is 2-D only")
        self.in_channels, self.out_channels, self.nb = in_channels, out_channels, nb
        cin = in_channels + 1  # noise-level channel
        conv = _CONV[dim][0]
        self.m_head = conv(cin, nc[0], 3, 1, 1, bias=False)
        self.m_down1 = _stage(nc[0], nc[1], nb, True, dim)
        self.m_down2 = _stage(nc[1], nc[2], nb, True, dim)
        self.m_down3 = _stage(nc[2], nc[3], nb, True, dim)
        self.m_body = nn.Sequential(*[ResBlock(nc[3], dim=dim) for _ in range(nb)])
        if dim == 3 and nb == 1:   # the reference's `sequential` unwraps a single module: its 3-D state_dict says m_body.res.*
            self.m_body = self.m_body[0]
        self.m_up3 = _stage(nc[3], nc[2], nb, False, dim)
        self.m_up2 = _stage(nc[2], nc[1], nb, False, dim)
        self.m_up1 = _stage(nc[1], nc[0], nb, False, dim)
        self.m_tail = conv(nc[0], out_channels, 3, 1, 1, bias=False)
        self.dim = dim
        self.precision = precision
        self._tc = None  # tensor-core engine (packed bf16 weights), built lazily
        self._tc32 = None  # fp32-grade tensor-core engine (packed tf32 hi/lo weights), built lazily
        if pretrained is not None:
            if pretrained.startswith("download"):
                raise RuntimeError("pretrained weights cannot be downloaded here (no network): pass a checkpoint path "
                                   "or pretrained=None and load a state_dict")
            self.load_state_dict(torch.load(pretrained, map_location="cpu"), strict=True)
            self.eval()
        else:
            self.apply(weights_init_drunet)
        if device is not None:
            self.to(device)

    # ---- fp32 path (CUDA-core kernels, matches the reference to ~1e-6) ---------------------------
    @staticmethod
    def _resblocks_f32(t, blocks):
        for rb in blocks:
            u = ops.conv_f32_ag(t, rb.res[0].weight, relu=True)
            t = ops.conv_f32_ag(u, rb.res[2].weight, res=t)
        return t

    def _forward_unet_f32(self, x0):
        nb = self.nb
        x1 = ops.conv_f32_ag(x0, self.m_head.weight)
        x2 = ops.conv_f32_ag(self._resblocks_f32(x1, list(self.m_down1)[:nb]), self.m_down1[nb].weight, kind=1)
        x3 = ops.conv_f32_ag(self._resblocks_f32(x2, list(self.m_down2)[:nb]), self.m_down2[nb].weight, kind=1)
        x4 = ops.conv_f32_ag(self._resblocks_f32(x3, list(self.m_down3)[:nb]), self.m_down3[nb].weight, kind=1)
        x = self._resblocks_f32(x4, list(self.m_body))
        x = self._resblocks_f32(ops.conv_f32_ag(x, self.m_up3[0].weight, kind=2, xadd=x4), list(self.m_up3)[1:])
        x = self._resblocks_f32(ops.conv_f32_ag(x, self.m_up2[0].weight, kind=2, xadd=x3), list(self.m_up2)[1:])
        x = self._resblocks_f32(ops.conv_f32_ag(x, self.m_up1[0].weight, kind=2, xadd=x2), list(self.m_up1)[1:])
        return ops.conv_f32_ag(x, self.m_tail.weight, xadd=x1)

    # ---- 3-D (NCDHW volumes, forward only) ---------------------------------------------------------
    @staticmethod
    def _resblocks3d_f32(t, blocks):
        for rb in blocks:
            u = ops.conv3d_f32(t, rb.res[0].weight, relu=True)
            t = ops.conv3d_f32(u, rb.res[2].weight, res=t)
        return t

    def _forward_unet3d_f32(self, x0):
        nb, rbs, conv = self.nb, self._resblocks3d_f32, ops.conv3d_f32
        x1 = conv(x0, self.m_head.weight)
        x2 = conv(rbs(x1, list(self.m_down1)[:nb]), self.m_down1[nb].weight, kind=1)
        x3 = conv(rbs(x2, list(self.m_down2)[:nb]), self.m_down2[nb].weight, kind=1)
        x4 = conv(rbs(x3, list(self.m_down3)[:nb]), self.m_down3[nb].weight, kind=1)
        x = rbs(x4, body_blocks(self))
        x = rbs(conv(x, self.m_up3[0].weight, kind=2, xadd=x4), list(self.m_up3)[1:])
        x = rbs(conv(x, self.m_up2[0].weight, kind=2, xadd=x3), list(self.m_up2)[1:])
        x = rbs(conv(x, self.m_up1[0].weight, kind=2, xadd=x2), list(self.m_up1)[1:])
        return conv(x, self.m_tail.weight, xadd=x1)

    def forward_unet(self, x0: torch.Tensor) -> torch.Tensor:
        if self.dim == 3:
            _no_grad_guard(f"DRUNet(dim=3, precision='{self.precision}')", x0, self.m_head.weight)
            if self.precision in ("tc32", "tc32h"):
                from .tc_engine import drunet3d_forward_tc32

                return drunet3d_forward_tc32(self, x0)
            if self.precision == "bf16":
                raise NotImplementedError("DRUNet(dim=3) runs at precision 'fp32', 'tc32' or 'tc32h'; the bf16 engine is 2-D only")
            return self._forward_unet3d_f32(x0)
        if self.precision == "bf16":
            _no_grad_guard("DRUNet(precision='bf16')", x0, self.m_head.weight)
            from .tc_engine import drunet_forward_bf16

            return drunet_forward_bf16(self, x0)
        if self.precision in ("tc32", "tc32h"):
            _no_grad_guard(f"DRUNet(precision='{self.precision}')", x0, self.m_head.weight)
            from .tc_engine import drunet_forward_tc32

            return drunet_forward_tc32(self, x0)
        return self._forward_unet_f32(x0)

    def forward(self, x: torch.Tensor, sigma) -> torch.Tensor:
        B, ones = x.size(0), [1] * self.dim
        if isinstance(sigma, torch.Tensor):
            if sigma.ndim > 0:
                if sigma.shape == (B, 1, *x.shape[2:]):
                    noise_level_map = sigma
                elif sigma.shape in [(B,), (B, 1, *ones)]:
                    noise_level_map = sigma.view(B, 1, *ones).expand(-1, 1, *x.shape[2:2 + self.dim])
                else:
                    raise ValueError(
                        "Incorrect shape, sigma should be of shape (1,), (batch_size,) or (batch_size, 1, height, width, "
                        f"(depth)), got {tuple(sigma.shape)}")
            else:
                noise_level_map = torch.ones((B, 1, *x.shape[2:]), device=x.device) * sigma.to(x.device)
        else:
            noise_level_map = torch.full((B, 1, *x.shape[2:]), sigma, device=x.device, dtype=x.dtype)
        x = torch.cat((x, noise_level_map.to(x.dtype)), 1)
        if all((s % 8 == 0 and s > 31) for s in x.shape[2:]):
            return self.forward_unet(x)
        if self.training or any(x.size(2 + i) < 64 for i in range(self.dim)):
            return _test_pad(self.forward_unet, x, modulo=16)
        if self.dim == 3:
            raise NotImplementedError(
                "test_onesplit is not implemented yet for 3D. Please pass images with spatial shape smaller than 64, or multiple "
                "of 8 and larger than 31 to DRUNet.")
        return _test_onesplit(self.forward_unet, x, refield=64)


def _test_pad(model, L, modulo=16):
    """replicate-pad every spatial axis to a multiple of `modulo`, run, crop (models/utils.py:49-61)"""
    spatial = L.shape[2:]
    pad = [int(np.ceil(s / modulo) * modulo - s) for s in spatial]
    E = model(torch.nn.functional.pad(L, tuple(v for p in reversed(pad) for v in (0, p)), mode="replicate"))
    return E[(...,) + tuple(slice(0, s) for s in spatial)]


def _test_onesplit(model, L, refield=32, sf=1):
    """four overlapping quadrants (models/utils.py:64-101)"""
    h, w = L.shape[-2:]
    top, bottom = slice(0, (h // 2 // refield + 1) * refield), slice(h - (h // 2 // refield + 1) * refield, h)
    left, right = slice(0, (w // 2 // refield + 1) * refield), slice(w - (w // 2 // refield + 1) * refield, w)
    Es = [model(L[..., a, b].contiguous()) for a, b in ((top, left), (top, right), (bottom, left), (bottom, right))]
    b, c = Es[0].shape[:2]
    E = torch.zeros(b, c, sf * h, sf * w, dtype=L.dtype, device=L.device)
    E[..., : h // 2 * sf, : w // 2 * sf] = Es[0][..., : h // 2 * sf, : w // 2 * sf]
    E[..., : h // 2 * sf, w // 2 * sf: w * sf] = Es[1][..., : h // 2 * sf, (-w + w // 2) * sf:]
    E[..., h // 2 * sf: h * sf, : w // 2 * sf] = Es[2][..., (-h + h // 2) * sf:, : w // 2 * sf]
    E[..., h // 2 * sf: h * sf, w // 2 * sf: w * sf] = Es[3][..., (-h + h // 2) * sf:, (-w + w // 2) * sf:]
    return E
