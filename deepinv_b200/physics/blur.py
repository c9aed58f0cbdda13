"""Blur (direct tiled convolution) and BlurFFT (spectral) on libdinvk kernels.

Drop-in for deepinv/physics/blur.py:443-737.  `Blur.A / A_adjoint` call `dinvk_blur_fwd / _adj`
(csrc/blur.cu: all five paddings resolved in index space, per-sample / per-channel filters as in
convolution.py:761-787), and `dinvk_blur3d_fwd / _adj` on (B,C,D,H,W) volumes; `use_fft=True` routes
the circular case through the spectral kernels.
`BlurFFT` keeps the reference's buffers (`filter`, `mask` = |h^| duplicated on a trailing axis, `angle`)
and its rfft2-domain U/V methods, but A / A_adjoint / A_adjoint_A / prox_l2 / A_dagger are single
fused launches of `dinvk_spectral` on PAIRS of real images packed as one complex image (a real
filter commutes with the packing), so a (B,C,H,W) batch costs B*C/2 complex 2-D transforms.
`SpaceVaryingBlur` (blur.py:740-868) is the product convolution sum_k h_k * (w_k . x) on one fused kernel per direction
(`dinvk_svblur_fwd / _adj`, csrc/blur.cu), and `TiledSpaceVaryingBlur` (blur.py:871-1192) its tiled form with one PSF per
overlapping patch (`dinvk_tiled_svblur_fwd / _adj`).
"""
from __future__ import annotations

import math
from warnings import warn

import torch
from torch import Tensor

from .. import _ffi, ops
from .forward import DecomposablePhysics, LinearPhysics, TensorKey, cache_hit, linear_apply


def _padding_code(padding: str) -> int:
    p = padding.lower()
    if p == "zeros":
        p = "constant"
    if p not in _ffi.PADDING_CODES:
        raise ValueError(f"padding = '{padding}' not implemented. Please use one of 'valid', 'circular', 'replicate', "
                         "'reflect', 'constant' or 'zeros'.")
    return _ffi.PADDING_CODES[p]


def _check_filter(filt: Tensor, B: int, C: int) -> None:
    b, c = filt.shape[:2]
    assert c in (1, C), f"Number of channels of the kernel is not matched for broadcasting, got c={c} and C={C}"
    assert b in (1, B), f"Batch size of the kernel is not matched for broadcasting, got b={b} and B={B}"


class Blur(LinearPhysics):
    r"""y = w * x (blur.py:443-561), on (B, C, H, W) images with (b, c, h, w) filters or on (B, C, D, H, W) volumes with
    (b, c, d, h, w) filters, b in {1, B}, c in {1, C}, all five paddings in both ranks.

    On volumes the direct kernel (`dinvk_blur3d_fwd / _adj`) runs for both values of ``use_fft``: the flag is stored as in
    the reference, where it selects FFT convolutions, the same operator up to rounding.  `A_dagger`, `prox_l2` and the norm
    estimate of a 3-D blur are the CG / power-method versions of LinearPhysics."""

    def __init__(self, filter: Tensor = None, padding: str = "valid", use_fft: bool = False, device="cpu", **kwargs):
        super().__init__(device=device, **kwargs)
        assert isinstance(filter, Tensor) or filter is None, \
            f"The filter must be a torch.Tensor or None, got filter of type {type(filter)}."
        self.padding = padding
        self.use_fft = use_fft
        self.register_buffer("filter", filter)
        self.to(device)

    def _fwd(self, x):
        return ops.blur_fwd(x, self.filter, _padding_code(self.padding))

    def A(self, x: Tensor, filter: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        if x.dim() == 5:
            return self._A3d(x)
        if x.dim() != 4:
            raise ValueError(f"Expected Tensor dimension to be 4 or 5, is {x.dim()}")
        if self.filter.dim() != 4:
            raise ValueError("Input and filter must be 4D tensors")
        _check_filter(self.filter, x.shape[0], x.shape[1])
        H, W = x.shape[-2:]
        code = _padding_code(self.padding)
        return linear_apply(x, self._fwd, lambda t: ops.blur_adj(t, self.filter, code, H, W))

    def A_adjoint(self, y: Tensor, filter: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        if y.dim() == 5:
            return self._At3d(y)
        if y.dim() != 4:
            raise ValueError(f"Expected Tensor dimension to be 4 or 5, is {y.dim()}")
        _check_filter(self.filter, y.shape[0], y.shape[1])
        code = _padding_code(self.padding)
        h, w = self.filter.shape[-2:]
        H, W = (y.shape[-2] + h - 1, y.shape[-1] + w - 1) if code == _ffi.PAD_VALID else y.shape[-2:]
        return linear_apply(y, lambda t: ops.blur_adj(t, self.filter, code, H, W), self._fwd)

    # 3-D: convolution.py:333-438 (conv3d / conv_transpose3d) on dinvk_blur3d_fwd / _adj
    def _filter3d(self, t: Tensor) -> int:
        if self.filter.dim() != 5:
            raise ValueError("Input and filter must be 5D tensors")
        _check_filter(self.filter, t.shape[0], t.shape[1])
        return _padding_code(self.padding)

    def _A3d(self, x: Tensor) -> Tensor:
        code = self._filter3d(x)
        D, H, W = x.shape[-3:]
        return linear_apply(x, lambda t: ops.blur3d_fwd(t, self.filter, code),
                            lambda t: ops.blur3d_adj(t, self.filter, code, D, H, W))

    def _At3d(self, y: Tensor) -> Tensor:
        code = self._filter3d(y)
        d, h, w = self.filter.shape[-3:]
        D, H, W = (y.shape[-3] + d - 1, y.shape[-2] + h - 1, y.shape[-1] + w - 1) if code == _ffi.PAD_VALID else y.shape[-3:]
        return linear_apply(y, lambda t: ops.blur3d_adj(t, self.filter, code, D, H, W),
                            lambda t: ops.blur3d_fwd(t, self.filter, code))

    def update_parameters(self, filter: Tensor = None, **kwargs):
        if filter is not None and self.filter is None:
            self.register_buffer("filter", filter)
            filter = None
        super().update_parameters(filter=filter, **kwargs)


class SpaceVaryingBlur(LinearPhysics):
    r"""y = sum_k h_k * (w_k . x), space-varying blur by product convolution (blur.py:740-868).

    :param torch.Tensor filters: h_k, (b, c, K, h, w) with b in {1, B}, c in {1, C}, h <= H and w <= W.
    :param torch.Tensor multipliers: w_k, (b, c, K, H, W), broadcast over (B, C) independently of the filters.
    :param str padding: 'valid', 'circular', 'replicate', 'reflect' or 'constant'.
    :param bool use_fft: stored as in the reference, where it selects FFT convolutions: the same operator up to rounding.
        Both values run the direct fused kernel here.

    `A` and `A_adjoint` take ``filters=``, ``multipliers=`` and ``padding=`` and store them; gradients flow to x only.
    `A_dagger`, `prox_l2` and the norm estimate are the CG / power-method versions of LinearPhysics."""

    def __init__(self, filters: Tensor = None, multipliers: Tensor = None, padding: str = "valid", use_fft: bool = False,
                 device="cpu", **kwargs):
        super().__init__(device=device, **kwargs)
        self.register_buffer("filters", filters)
        self.register_buffer("multipliers", multipliers)
        self.padding = padding
        self.use_fft = use_fft
        self.to(device)

    def A(self, x: Tensor, filters: Tensor = None, multipliers: Tensor = None, padding: str = None, **kwargs) -> Tensor:
        from . import functional as dF

        self.update_parameters(filters, multipliers, padding, **kwargs)
        return dF.product_convolution2d(x, self.multipliers, self.filters, self.padding, use_fft=self.use_fft)

    def A_adjoint(self, y: Tensor, filters: Tensor = None, multipliers: Tensor = None, padding: str = None, **kwargs) -> Tensor:
        from . import functional as dF

        self.update_parameters(filters=filters, multipliers=multipliers, padding=padding, **kwargs)
        return dF.product_convolution2d_adjoint(y, self.multipliers, self.filters, self.padding, use_fft=self.use_fft)

    def update_parameters(self, filters: Tensor = None, multipliers: Tensor = None, padding: str = None, **kwargs):
        if padding is not None:
            self.padding = padding
        super().update_parameters(filters=filters, multipliers=multipliers, **kwargs)


class TiledSpaceVaryingBlur(LinearPhysics):
    r"""y = sum_k Wt_k . (h_k * x), space-varying blur by tiled product convolution (blur.py:871-1192): one PSF per
    overlapping patch, blended by a partition of unity, valid padding.

    :param torch.Tensor filters: h_k, (b, c, K, h, w) with b in {1, B}, c in {1, C}; K = nr * nc patches, row-major.
    :param int, tuple[int, int] patch_size: patch (P1, P2).
    :param int, tuple[int, int] stride: stride (s1, s2) <= patch; defaults to half the patch.
    :param str blending_mode: 'bump' or 'linear' (`functional.generate_tiled_multipliers`).
    :param bool use_fft: stored as in the reference, where it selects FFT convolutions: the same operator up to rounding.
        Both values run the direct fused kernel here.

    The image is padded at the bottom / right to the compatible size that nr x nc patches tile; a patch reaching into that
    padding still counts where it overlaps the image.  `A` and `A_adjoint` take ``filters=`` and store them; the multipliers
    (buffer `multipliers`, (1, 1, K, P1, P2)) are regenerated only when the image size changes.  One fused kernel per direction
    (`dinvk_tiled_svblur_fwd / _adj`); gradients flow to x only.  `A_dagger`, `prox_l2` and the norm estimate are the CG /
    power-method versions of LinearPhysics."""

    def __init__(self, filters: Tensor = None, patch_size=None, stride=None, blending_mode: str = "bump", use_fft: bool = True,
                 device="cpu", dtype=torch.float32, **kwargs):
        from .functional import _resolve_tiling_params

        super().__init__(device=device, **kwargs)
        self.patch_size, self.stride = _resolve_tiling_params(patch_size, stride)
        self.pad_if_needed = True
        self.blending_mode = blending_mode
        self.use_fft = use_fft
        self._dynamic_img_size = None
        self.register_buffer("filters", filters)
        self.register_buffer("multipliers", None)
        self.to(device=device, dtype=dtype)

    @staticmethod
    def num_filters(img_size, patch_size, stride=None) -> tuple[int, int]:
        """patches (nr, nc) along each dimension, hence the number of filters nr * nc, for an image of `img_size`"""
        from .functional import _as_pair, _num_patches, _resolve_tiling_params

        return _num_patches(_as_pair(img_size), *_resolve_tiling_params(patch_size, stride))

    def get_num_patches(self, img_size) -> tuple[int, int]:
        from .functional import _as_pair, _num_patches

        return _num_patches(_as_pair(img_size), self.patch_size, self.stride)

    def get_needed_pad(self, img_size) -> tuple[int, int]:
        from .functional import _as_pair, _needed_pad

        return _needed_pad(_as_pair(img_size), self.patch_size, self.stride)

    def get_compatible_img_size(self, img_size) -> tuple[int, int]:
        from .functional import _as_pair, _compatible_size

        return _compatible_size(_as_pair(img_size), self.patch_size, self.stride)

    def _operands(self, t: Tensor, H: int, W: int):
        """the reference's failure modes on an (H, W) image"""
        h, w = self.filters, self.multipliers
        nr, nc = self.get_num_patches((H, W))
        if nr * nc != h.size(2):
            raise ValueError(f"The total number of patches must be equal to the number of PSFs, got {nr * nc} and {h.size(2)}")
        if tuple(w.shape) != (1, 1, nr * nc, *self.patch_size):
            raise NotImplementedError(f"multipliers of shape {tuple(w.shape)}: only the shared (1, 1, K, P1, P2) blending of "
                                      "generate_tiled_multipliers is supported")
        if t.dim() != 4:
            raise ValueError(f"Input image must have shape (B, C, H, W), got {tuple(t.shape)}.")
        _check_filter(h, t.size(0), t.size(1))
        return w, h

    def A(self, x: Tensor, filters: Tensor = None, **kwargs) -> Tensor:
        H, W = x.shape[-2:]
        self.update_parameters(filters, img_size=(H, W), device=x.device, **kwargs)
        w, h = self._operands(x, H, W)
        return linear_apply(x, lambda t: ops.tiled_svblur_fwd(t, w, h, self.stride),
                            lambda t: ops.tiled_svblur_adj(t, w, h, self.stride, H, W))

    def A_adjoint(self, y: Tensor, filters: Tensor = None, **kwargs) -> Tensor:
        # valid padding: the image is the measurement grown by the filter
        fh, fw = (self.filters if filters is None else filters).shape[-2:]
        H, W = y.shape[-2] + fh - 1, y.shape[-1] + fw - 1
        self.update_parameters(filters, img_size=(H, W), device=y.device, **kwargs)
        w, h = self._operands(y, H, W)
        return linear_apply(y, lambda t: ops.tiled_svblur_adj(t, w, h, self.stride, H, W),
                            lambda t: ops.tiled_svblur_fwd(t, w, h, self.stride))

    def update_parameters(self, filters: Tensor = None, img_size=None, device=None, **kwargs):
        from .functional import generate_tiled_multipliers

        if isinstance(filters, Tensor):
            self.register_buffer("filters", filters.to(device) if device is not None else filters)
        if img_size is not None and (self.multipliers is None or tuple(img_size) != self._dynamic_img_size
                                     or (device is not None and self.multipliers.device != torch.device(device))):
            w = generate_tiled_multipliers(self.get_compatible_img_size(img_size), self.patch_size, self.stride,
                                           mode=self.blending_mode, device=device if device is not None else "cpu")
            self.register_buffer("multipliers", w)
            self._dynamic_img_size = tuple(img_size)
        super().update_parameters(**kwargs)


class BlurFFT(DecomposablePhysics):
    r"""circular blur diagonalised by the 2-D DFT (blur.py:564-737)"""

    def __init__(self, img_size: tuple, filter: Tensor | None = None, device="cpu", **kwargs):
        super().__init__(device=device, **kwargs)
        self.img_size = tuple(img_size)
        assert isinstance(filter, Tensor) or filter is None, \
            f"The filter must be a torch.Tensor or None, got filter of type {type(filter)}."
        self._spec_key = None
        params = self.get_filter_parameters(self.img_size, filter, device)
        self.register_buffer("filter", params["filter"])
        self.register_buffer("angle", params["angle"])
        self.register_buffer("mask", params["mask"])
        self.to(device)

    # ---- parameters (blur.py:659-737) ---------------------------------------------------------------
    @staticmethod
    def _full_spectrum(filt: Tensor, img_size) -> Tensor:
        """un-normalised 2-D DFT of the zero-padded, centre-rolled filter (convolution.py:790-812), full (C,H,W)
        complex spectrum, computed with the library's own transform"""
        H, W = img_size[-2:]
        h, w = filt.shape[-2:]
        f = torch.nn.functional.pad(filt.float(), (0, W - w, 0, H - h))
        f = torch.roll(f, shifts=(-int(h / 2), -int(w / 2)), dims=(-2, -1))
        n = f.shape[0] * f.shape[1]
        planar = torch.stack([f.reshape(n, H, W), torch.zeros(n, H, W, device=f.device)], 1)
        spec = ops.spectral(planar, H, W, fwd=True, inv=False, centered=False) * math.sqrt(H * W)
        return torch.complex(spec[:, 0], spec[:, 1]).reshape(f.shape[0], f.shape[1], H, W)

    @staticmethod
    def get_filter_parameters(img_size, filter, device="cpu") -> dict:
        if filter is None or not isinstance(filter, Tensor):
            return {"filter": None, "angle": None, "mask": None}
        filter = filter.to(device)
        if img_size[0] > filter.shape[1]:
            filter = filter.repeat(1, img_size[0], 1, 1)
        full = BlurFFT._full_spectrum(filter, img_size)
        half = full[..., : img_size[-1] // 2 + 1]
        mag = torch.abs(half)
        angle = torch.exp(1.0j * torch.angle(half))
        m = mag.unsqueeze(-1)
        return {"filter": filter, "angle": angle, "mask": torch.cat([m, m], dim=-1)}

    def update_parameters(self, filter: Tensor | None = None, **kwargs):
        if filter is not None:
            dev = self.filter.device if isinstance(self.filter, Tensor) else filter.device
            if isinstance(self.filter, Tensor) and self.filter.device != filter.device:
                warn("The provided ``filter`` is on a different device than the current filter ``self.filter``. "
                     f"The current underlying self.filter.device={self.filter.device} will be used.", stacklevel=2)
            params = self.get_filter_parameters(self.img_size, filter, dev)
            for k, v in params.items():
                if getattr(self, k, None) is None:
                    self.register_buffer(k, v)
                else:
                    setattr(self, k, v)
        if kwargs.get("mask") is None and "mask" in kwargs:
            kwargs.pop("mask")
        super().update_parameters(**kwargs)

    # ---- device-side multipliers derived from (mask, angle) -------------------------------------------
    def _mult(self):
        m, a = self.mask, self.angle
        if not cache_hit(self._spec_key, m, a):
            H, W = self.img_size[-2:]
            half = m[..., 0] * a                       # h^ on the half spectrum (Fb, C, H, W/2+1), Fb = 1 or one filter per sample
            Fb, C = half.shape[:2]
            same = Fb == 1 and (C == 1 or bool((half == half[:, :1]).all()))
            hh = half[:, :1] if same else half
            # Hermitian completion: h^[k1, k2] = conj(h^[-k1, W-k2]) for k2 > W/2
            k2 = torch.arange(W // 2 + 1, W, device=m.device)
            src = torch.roll(torch.flip(hh, dims=(-2,)), 1, dims=-2)[..., W - k2]
            full = torch.cat([hh, torch.conj(src)], dim=-1).contiguous()  # (Fb, C', H, W); the batch dimension is KEPT
            if same:
                full = full[0]
            mag = full.abs()
            pinv = torch.where(mag > 1e-5, 1.0 / mag, torch.zeros_like(mag))
            ang = torch.where(mag > 0, full / mag.clamp_min(1e-38), torch.ones_like(full))
            self._h = ops.MaskSpec(torch.view_as_real(full).contiguous(), H * W if not same else 0, 0, W, True)
            self._hdag = ops.MaskSpec(torch.view_as_real(torch.conj(ang) * pinv).contiguous(), H * W if not same else 0, 0, W, True)
            self._habs = ops.MaskSpec(mag.contiguous(), H * W if not same else 0, 0, W, False)
            self._same = same
            self._spec_key = TensorKey(m, a)
        return self._h, self._hdag, self._habs, self._same

    # ---- packing of real images into complex ones --------------------------------------------------------
    def _run(self, x: Tensor, gmode, spec, p1=None, a1=0.0, c=0.0) -> Tensor:
        B, C, H, W = x.shape
        _, _, _, same = self._mult()
        x = x.float().contiguous()
        n = B * C
        if same:
            xs = [x] if p1 is None else [x, p1.float().contiguous()]
            if n % 2:
                xs = [torch.cat([t.reshape(n, H, W), torch.zeros(1, H, W, device=x.device)], 0) for t in xs]
            planar = [t.reshape(-1, 2, H, W) for t in xs]
            out = ops.spectral(planar[0], H, W, fwd=True, inv=True, centered=False, gmode=gmode, mask=spec,
                               p1=planar[1] if p1 is not None else None, a1=a1, c=c)
            return out.reshape(-1, H, W)[:n].reshape(B, C, H, W)
        # per-channel filters: one complex image per real image (imaginary plane zero), multiplier per image
        z = torch.zeros(n, 2, H, W, device=x.device)
        z[:, 0] = x.reshape(n, H, W)
        z1 = None
        if p1 is not None:
            z1 = torch.zeros(n, 2, H, W, device=x.device)
            z1[:, 0] = p1.float().reshape(n, H, W)
        # per-sample and / or per-channel filters (the reference broadcasts a (Fb, C', H, W/2+1, 2) mask over the batch,
        # blur.py:659-692 + forward.py:1080-1116): one multiplier per (sample, channel) image
        t = spec.tensor                                     # (Fb, C', H, W[, 2])
        Fb, Cf = t.shape[:2]
        if Fb not in (1, B) or Cf not in (1, C):
            raise RuntimeError(f"BlurFFT: filter spectrum of shape {tuple(t.shape[:2])} does not broadcast to a batch of {B} x {C} images")
        exp = t.expand(B, C, *t.shape[2:]).reshape(n, *t.shape[2:]).contiguous()
        spec_b = ops.MaskSpec(exp, H * W, 0, W, spec.complex)
        out = ops.spectral(z, H, W, fwd=True, inv=True, centered=False, gmode=gmode, mask=spec_b, p1=z1, a1=a1, c=c)
        return out[:, 0].reshape(B, C, H, W)

    def _checkx(self, x):
        if x.dim() != 4 or tuple(x.shape[-2:]) != tuple(self.img_size[-2:]):
            raise ValueError(f"expected a (B,C,{self.img_size[-2]},{self.img_size[-1]}) tensor, got {tuple(x.shape)}")

    def A(self, x: Tensor, filter: Tensor | None = None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        self._checkx(x)
        h, _, _, _ = self._mult()
        f = lambda t: self._run(t, _ffi.G_CMUL, h)
        g = lambda t: self._run(t, _ffi.G_CMUL_CONJ, h)
        return linear_apply(x, f, g)

    def A_adjoint(self, y: Tensor, filter: Tensor | None = None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        self._checkx(y)
        h, _, _, _ = self._mult()
        f = lambda t: self._run(t, _ffi.G_CMUL, h)
        g = lambda t: self._run(t, _ffi.G_CMUL_CONJ, h)
        return linear_apply(y, g, f)

    def A_adjoint_A(self, x: Tensor, filter=None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        self._checkx(x)
        _, _, habs, _ = self._mult()
        f = lambda t: self._run(t, _ffi.G_SQ, habs)
        return linear_apply(x, f, f)

    def A_A_adjoint(self, y: Tensor, filter=None, **kwargs) -> Tensor:
        return self.A_adjoint_A(y, filter=filter, **kwargs)  # U unitary, real diagonal: same operator

    def prox_l2(self, z: Tensor, y: Tensor, gamma, **kwargs) -> Tensor:
        needs_grad = torch.is_grad_enabled() and (z.requires_grad or y.requires_grad or
                                                  (isinstance(gamma, Tensor) and gamma.requires_grad))
        if needs_grad or (isinstance(gamma, Tensor) and gamma.numel() > 1):
            return super().prox_l2(z, y, gamma, **kwargs)
        self._checkx(z)
        h, _, habs, _ = self._mult()
        g = float(gamma)
        aty = self._run(y, _ffi.G_CMUL_CONJ, h)
        return self._run(aty, _ffi.G_INV_SQ_PLUS_C, habs, p1=z, a1=1.0 / g, c=1.0 / g)

    def A_dagger(self, y: Tensor, filter=None, **kwargs) -> Tensor:
        self.update_parameters(filter=filter, **kwargs)
        if torch.is_grad_enabled() and y.requires_grad:
            return super().A_dagger(y)
        self._checkx(y)
        _, hdag, _, _ = self._mult()
        return self._run(y, _ffi.G_CMUL, hdag)

    # ---- rfft2-domain factors of the SVD (blur.py:639-657), needed by DDRM ---------------------------------
    def _rfft2(self, x: Tensor) -> Tensor:
        B, C, H, W = x.shape
        z = torch.zeros(B * C, 2, H, W, device=x.device)
        z[:, 0] = x.float().reshape(B * C, H, W)
        s = ops.spectral(z, H, W, fwd=True, inv=False, centered=False)
        return torch.complex(s[:, 0], s[:, 1])[..., : W // 2 + 1].reshape(B, C, H, W // 2 + 1)

    def _irfft2(self, xh: Tensor) -> Tensor:
        B, C, H, Wh = xh.shape
        W = self.img_size[-1]
        # irfft2 semantics: the imaginary parts of the self-conjugate bins are ignored
        k2 = torch.arange(W // 2 + 1, W, device=xh.device)
        src = torch.roll(torch.flip(xh, dims=(-2,)), 1, dims=-2)[..., W - k2]
        full = torch.cat([xh, torch.conj(src)], dim=-1)
        z = torch.stack([full.real, full.imag], 2).reshape(B * C, 2, H, W).contiguous().float()
        s = ops.spectral(z, H, W, fwd=False, inv=True, centered=False)
        return s[:, 0].reshape(B, C, H, W)  # real part == c2r semantics (imaginary residue of the k2=0, W/2 columns dropped)

    def V_adjoint(self, x: Tensor) -> Tensor:
        return torch.view_as_real(self._rfft2(x))

    def V(self, x: Tensor, **kwargs) -> Tensor:
        return self._irfft2(torch.view_as_complex(x.contiguous()))

    def U(self, x: Tensor) -> Tensor:
        return self._irfft2(torch.view_as_complex(x.contiguous()) * self.angle)

    def U_adjoint(self, x: Tensor, **kwargs) -> Tensor:
        return torch.view_as_real(self._rfft2(x) * torch.conj(self.angle))


class Downsampling(LinearPhysics):
    r"""y = S_f (h * x): anti-aliasing blur followed by decimation by `factor` (deepinv/physics/blur.py:15-440).

    `A` is the tiled correlation kernel (`dinvk_blur_fwd`) followed by the strided pick, `A_adjoint` the zero-stuffed
    upsampling followed by the exact transposed kernel (`dinvk_blur_adj`), for all five paddings.  With circular padding
    `prox_l2` is the closed form of Zhao et al. (blur.py:332-364): the f x f aliasing fold of |h^|^2 is inverted bin by
    bin; the two 2-D transforms run on the library's spectral kernel (`dinvk_spectral`, un-centred), the fold itself is
    a handful of elementwise passes on the spectrum.  Other paddings: CG on the operator kernels (LinearPhysics)."""

    def __init__(self, img_size=None, filter="warn", factor: int = 2, device="cpu", padding: str = "circular", **kwargs):
        if isinstance(filter, str) and filter == "warn":
            warn("Leaving the filter as default is deprecated and will be removed in future versions. Please specify "
                 "filter=None for bare decimation, or one of the available filters (gaussian, bilinear, bicubic, sinc).",
                 stacklevel=2)
            filter = None
        super().__init__(device=device, **kwargs)
        self.imsize = tuple(img_size) if isinstance(img_size, list) else img_size
        self.imsize_dynamic = (3, 128, 128)
        self.padding = padding
        _padding_code(padding)
        self.factor = self.check_factor(factor)
        self.register_buffer("filter", self._make_filter(filter, self.factor, device))
        self._fh_key = None
        self.to(device)

    @staticmethod
    def check_factor(factor) -> int:
        if isinstance(factor, (int, float)):
            return int(factor)
        if isinstance(factor, Tensor):
            if factor.ndim > 1:
                raise ValueError("Factor tensor must be 1D.")
            u = torch.unique(factor)
            if len(u) > 1:
                raise ValueError(f"Downsampling only supports one unique factor per batch, but got factors {u.tolist()}.")
            return int(u.item())
        raise ValueError(f"Factor must be an int, float or a 1D Tensor, got {type(factor)}.")

    @staticmethod
    def _make_filter(filter, factor, device):
        from . import functional as dF

        if filter is None:
            return None
        if isinstance(filter, list):
            if len(set(filter)) == 1 and isinstance(filter[0], str):
                filter = filter[0]
            else:
                raise ValueError("Downsampling supports filter string lists if they are identical, but got unique filters "
                                 f"{set(filter)}.")
        if isinstance(filter, Tensor):
            return filter.to(device)
        if filter == "gaussian":
            return dF.gaussian_blur(sigma=(factor, factor), device=device)
        if filter == "bilinear":
            return dF.bilinear_filter(factor, device=device)
        if filter == "bicubic":
            return dF.bicubic_filter(factor, device=device)
        if filter == "sinc":
            return dF.sinc_filter(factor, length=4 * factor, device=device)
        raise ValueError(f"unknown filter {filter!r}")

    def update_parameters(self, filter=None, factor=None, **kwargs):
        if factor is not None:
            if filter is None and self.filter is not None:
                warn("Updating factor but not filter. Filter will not be valid for new factor. Pass filter string or new "
                     "filter to resolve this.")
            self.factor = self.check_factor(factor)
        if filter is not None:
            dev = self.filter.device if isinstance(self.filter, Tensor) else \
                (filter.device if isinstance(filter, Tensor) else kwargs.get("device", "cpu"))
            f = self._make_filter(filter, self.factor, dev)
            if self.filter is None:
                self.register_buffer("filter", f)
            else:
                self.filter = f.to(self.filter.device)
        kwargs.pop("device", None)
        super().update_parameters(**kwargs)

    # ---- operator -------------------------------------------------------------------------------------------
    def _blur(self, x):
        return x if self.filter is None else ops.blur_fwd(x, self.filter, _padding_code(self.padding))

    def _blur_t(self, v, H, W):
        return v if self.filter is None else ops.blur_adj(v, self.filter, _padding_code(self.padding), H, W)

    def _down(self, x):
        f = self.factor
        return self._blur(x)[:, :, ::f, ::f].contiguous()

    def _up(self, y, H, W):
        """A^T: zero-stuffing to the blurred image's size (H', W'), then the transposed blur back to (H, W)"""
        f = self.factor
        valid = self.filter is not None and _padding_code(self.padding) == _ffi.PAD_VALID
        Hb, Wb = (H - self.filter.shape[-2] + 1, W - self.filter.shape[-1] + 1) if valid else (H, W)
        v = torch.zeros(y.shape[0], y.shape[1], Hb, Wb, device=y.device, dtype=torch.float32)
        v[:, :, ::f, ::f] = y
        return self._blur_t(v, H, W)

    def A(self, x: Tensor, filter=None, factor=None, **kwargs) -> Tensor:
        self.imsize_dynamic = tuple(x.shape[-3:])
        self.update_parameters(filter=filter, factor=factor, device=x.device, **kwargs)
        if x.dim() != 4:
            raise ValueError(f"Expected Tensor dimension to be 4, is {x.dim()}")
        if self.filter is not None:
            _check_filter(self.filter, x.shape[0], x.shape[1])
        H, W = x.shape[-2:]
        return linear_apply(x, self._down, lambda t: self._up(t, H, W))

    def A_adjoint(self, y: Tensor, filter=None, factor=None, **kwargs) -> Tensor:
        f = self.check_factor(factor) if factor is not None else self.factor
        self.imsize_dynamic = (y.shape[-3], y.shape[-2] * f, y.shape[-1] * f)
        self.update_parameters(filter=filter, factor=factor, device=y.device, **kwargs)
        imsize = self.imsize if self.imsize is not None else self.imsize_dynamic
        H, W = imsize[-2:]
        return linear_apply(y, lambda t: self._up(t, H, W), self._down)

    # ---- closed-form prox for circular padding ------------------------------------------------------------------
    def _spectrum(self, C, H, W):
        """F h (un-normalised 2-D DFT of the zero-padded, centre-rolled filter): (1|B, C, H, W) complex"""
        f = self.filter
        if not cache_hit(self._fh_key, f, extra=(C, H, W)):
            ff = f if f.shape[1] == C else f.expand(f.shape[0], C, *f.shape[-2:])
            self._Fh = BlurFFT._full_spectrum(ff, (C, H, W))
            self._fh_key = TensorKey(f, extra=(C, H, W))
        return self._Fh

    def prox_l2(self, z: Tensor, y: Tensor, gamma, use_fft: bool = True, **kwargs) -> Tensor:
        tracked = torch.is_grad_enabled() and (z.requires_grad or y.requires_grad or
                                               (isinstance(gamma, Tensor) and gamma.requires_grad))
        if not (use_fft and self.padding == "circular" and self.filter is not None) or tracked or \
                (isinstance(gamma, Tensor) and gamma.numel() > 1):
            return LinearPhysics.prox_l2(self, z, y, gamma, **kwargs)
        g = float(gamma)
        B, C, H, W = z.shape
        sf = self.factor
        z_hat = ops.axpbypcz(self.A_adjoint(y), 1.0, z, 1.0 / g)
        planar = torch.zeros(B * C, 2, H, W, device=z.device)
        planar[:, 0] = z_hat.reshape(B * C, H, W)
        s = ops.spectral(planar, H, W, fwd=True, inv=False, centered=False)  # orthonormal: linear, undone by the inverse
        Fz = torch.complex(s[:, 0], s[:, 1]).reshape(B, C, H, W)
        Fh = self._spectrum(C, H, W)

        def fold(a):  # mean over the sf x sf aliases: (.., H, W) -> (.., H/sf, W/sf)
            return a.reshape(*a.shape[:-2], sf, H // sf, sf, W // sf).mean(dim=(-4, -2))

        top = fold(Fh * Fz)
        below = fold((Fh.conj() * Fh).real) + 1.0 / g
        rc = Fh.conj() * (top / below).repeat(1, 1, sf, sf)
        rp = torch.stack([rc.real, rc.imag], 2).reshape(B * C, 2, H, W).contiguous()
        r = ops.spectral(rp, H, W, fwd=False, inv=True, centered=False)[:, 0].reshape(B, C, H, W)
        return ops.axpbypcz(z_hat, g, r, -g)


class Upsampling(Downsampling):
    r"""x = h^T * S^T (y): the transpose of `Downsampling` used as the forward operator (blur.py:392-440).  `A` is
    Downsampling.A_adjoint and `A_adjoint` is Downsampling.A, on the same kernels; ``img_size`` is the (C, H, W) of the
    upsampled image."""

    def __init__(self, img_size, filter=None, factor: int = 2, padding: str = "circular", device="cpu", **kwargs):
        assert padding != "valid", "Padding 'valid' is not supported for Upsampling operator."
        super().__init__(img_size=img_size, filter=filter, factor=factor, padding=padding, device=device, **kwargs)

    def A(self, x: Tensor, **kwargs) -> Tensor:
        return super().A_adjoint(x, **kwargs)

    def A_adjoint(self, y: Tensor, **kwargs) -> Tensor:
        return super().A(y, **kwargs)

    def prox_l2(self, z: Tensor, y: Tensor, gamma, use_fft: bool = True, **kwargs) -> Tensor:
        # Downsampling's closed form with the roles swapped: the reference multiplies the spectrum of the (C, H, W) image size
        # by that of z, which lives on the small grid, and fails on the size mismatch
        if use_fft and self.padding == "circular" and self.filter is not None:
            H, W = self.imsize[-2:]
            if tuple(z.shape[-2:]) != (H, W):
                dim = 3 if z.shape[-1] != W else 2
                raise RuntimeError(f"The size of tensor a ({(H, W)[dim - 2]}) must match the size of tensor b "
                                   f"({z.shape[dim]}) at non-singleton dimension {dim}")
        return super().prox_l2(z, y, gamma, use_fft=use_fft, **kwargs)


class DownsamplingMatlab(Downsampling):
    r"""MATLAB ``imresize(x, 1 / factor, 'bicubic')``: the antialiased cubic kernel with reflect padding (blur.py:1195-1261).

    `A` is one launch of the fused separable resize (`dinvk_resize_fwd`, csrc/blur.cu) and `A_adjoint` one launch of its exact
    transpose (`dinvk_resize_adj`) on the (H_out f, W_out f) image, the domain on which the reference's autograd adjoint
    lives.  The factor is truncated to an int as `Downsampling.check_factor` does, so a factor below 2 is the identity.
    `A` is differentiable in x through the transpose kernel and `A_adjoint` in y through the forward kernel.  `prox_l2`,
    `A_dagger` and the norm estimate are the inherited CG / power-method versions (reflect padding)."""

    def __init__(self, factor=2, kernel: str = "cubic", padding: str = "reflect", antialiasing: bool = True, device="cpu",
                 **kwargs):
        super().__init__(filter=None, factor=factor, device=device, **kwargs)
        self.kernel = kernel
        self.padding = padding
        self.antialiasing = antialiasing

    def _plan(self, H: int, W: int):
        from .imresize import resize_plan

        return resize_plan(H, W, scale=1 / self.factor, antialiasing=self.antialiasing, kernel=self.kernel,
                           padding_type=self.padding)

    def A(self, x: Tensor, factor=None, **kwargs) -> Tensor:
        from .imresize import resize

        self.update_parameters(factor=factor, device=x.device, **kwargs)
        if x.dim() not in (2, 3, 4):
            raise ValueError("{}-dim Tensor is not supported!".format(x.dim()))
        h, w = x.shape[-2:]
        out, th, tw = self._plan(h, w)
        if th is None and tw is None:
            return x.clone()
        return resize(x.reshape(-1, 1, h, w), th, tw).reshape(*x.shape[:-2], *out)

    def A_adjoint(self, y: Tensor, factor=None, **kwargs) -> Tensor:
        from .imresize import resize_adjoint

        self.update_parameters(factor=factor, device=y.device, **kwargs)
        if y.dim() != 4:
            raise ValueError(f"Expected Tensor dimension to be 4, is {y.dim()}")
        H, W = y.shape[-2] * self.factor, y.shape[-1] * self.factor
        _, th, tw = self._plan(H, W)
        return y.clone() if th is None and tw is None else resize_adjoint(y, th, tw, H, W)

    def prox_l2(self, z: Tensor, y: Tensor, gamma, use_fft: bool = True, **kwargs) -> Tensor:
        # reflect padding: the inherited CG route, which starts from A^T y + z / gamma.  A^T y lives on the (H_out f, W_out f)
        # grid, so, as in the reference, an image whose sides are not multiples of the factor does not broadcast against it
        if isinstance(z, Tensor):
            torch.broadcast_shapes(tuple(z.shape), (*y.shape[:-2], y.shape[-2] * self.factor, y.shape[-1] * self.factor))
        return super().prox_l2(z, y, gamma, use_fft=use_fft, **kwargs)
