"""MRI / MultiCoilMRI on the fused sm_90a spectral kernels.

Drop-in for deepinv/physics/mri.py:11-695 (2-D and 2-D+t: MRI, MultiCoilMRI, DynamicMRI, SequentialMRI; `three_d=True`
volumes for MRI and MultiCoilMRI).  Same constructor, buffers (`mask`, `coil_maps`), kwargs-store-as-buffer side effects and
error types.  Every method below is one call of `dinvk_spectral` or, on (B,2,D,H,W) volumes, of `dinvk_spectral3d`
(csrc/spectral.cu); nothing is computed with torch.fft and no volume is permuted.
"""
from __future__ import annotations

from warnings import warn

import numpy as np
import torch
from torch import Tensor

from .. import _ffi, ops
from .forward import DecomposablePhysics, LinearPhysics, TensorKey, cache_hit, linear_apply


class MRIMixin:
    """mask / layout helpers (deepinv/utils/mixins.py:118-287)"""

    @staticmethod
    def check_mask(mask: Tensor = None, three_d: bool = False, **kwargs) -> Tensor:
        if mask is not None:
            if isinstance(mask, np.ndarray):
                mask = torch.from_numpy(mask)
            while len(mask.shape) < (4 if not three_d else 5):
                mask = mask.unsqueeze(0)
            if mask.shape[1] == 1:
                mask = torch.cat([mask, mask], dim=1)
        return mask

    @staticmethod
    def to_torch_complex(x: Tensor) -> Tensor:
        return torch.view_as_complex(x.moveaxis(1, -1).contiguous())

    @staticmethod
    def from_torch_complex(x: Tensor) -> Tensor:
        return torch.view_as_real(x).moveaxis(-1, 1)

    # centred orthonormal 2-D (three_d: 3-D) DFT on planar (B,2,H,W) / (B,2,D,H,W) tensors (mixins.py:158-206)
    def im_to_kspace(self, x: Tensor, three_d: bool = False) -> Tensor:
        return linear_apply(x, lambda t: _dft(t, three_d, False), lambda t: _dft(t, three_d, True))

    def kspace_to_im(self, y: Tensor, three_d: bool = False) -> Tensor:
        return linear_apply(y, lambda t: _dft(t, three_d, True), lambda t: _dft(t, three_d, False))

    def crop(self, x: Tensor, crop: bool = True, shape=None, rescale: bool = False) -> Tensor:
        """centre crop to img_size (mixins.py:208-247)"""
        crop_size = tuple(shape[-2:]) if shape is not None else tuple(self.img_size[-2:])
        odd_h = crop_size[0] % 2 == 1
        if odd_h:
            crop_size = (crop_size[0] + 1, crop_size[1])
        if rescale and crop:
            raise ValueError("Only one of rescale or crop can be used.")
        if rescale:
            out = torch.nn.functional.interpolate(x.reshape(-1, 1, *x.shape[-2:]), size=crop_size, mode="bilinear",
                                                  antialias=True).reshape(*x.shape[:-2], *crop_size)
        elif crop:
            h, w = x.shape[-2:]
            ph, pw = max(crop_size[0] - h, 0), max(crop_size[1] - w, 0)
            if ph or pw:  # torchvision's CenterCrop zero-pads an input smaller than the crop (the smaller half on top / left)
                x = torch.nn.functional.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
                h, w = x.shape[-2:]
            top = int(round((h - crop_size[0]) / 2.0))
            left = int(round((w - crop_size[1]) / 2.0))
            out = x[..., top: top + crop_size[0], left: left + crop_size[1]]
        else:
            return x
        return out[..., :-1, :] if odd_h else out

    @staticmethod
    def rss(x: Tensor, multicoil: bool = True, mag: bool = True, three_d: bool = False) -> Tensor:
        if x.shape[1] != 2 or x.is_complex():
            raise ValueError("x should be of shape (B,2,...) and not of complex dtype.")
        ss = x.pow(2)
        if mag:
            ss = ss.sum(dim=1, keepdim=True)
        if multicoil:
            ss = ss.sum(dim=2)
        return ss.sqrt()


def _dft(t: Tensor, three_d: bool, inverse: bool) -> Tensor:
    """centred orthonormal DFT over the last two (three_d: three) dims of a planar (B,2,...) tensor"""
    if three_d:
        if t.dim() < 5 or t.shape[1] != 2:
            raise ValueError(f"expected a planar (B,2,...,D,H,W) tensor, got {tuple(t.shape)}")
        return ops.spectral3d(t, *t.shape[-3:], fwd=not inverse, inv=inverse)
    return ops.spectral(t, *t.shape[-2:], fwd=not inverse, inv=inverse)


class _MaskCache:
    """device-side multiplier description derived from the `mask` buffer; rebuilt when the buffer changes"""

    def __init__(self):
        self.key = None
        self.spec = None

    def get(self, mask: Tensor, three_d: bool = False) -> ops.MaskSpec:
        if not cache_hit(self.key, mask):
            self.spec = ops.mask_spec3d(mask) if three_d else ops.mask_spec_from_real(mask, mask.shape[-2], mask.shape[-1])
            self.key = TensorKey(mask)
        return self.spec


class MRI(MRIMixin, DecomposablePhysics):
    r"""Single-coil accelerated MRI y = M F x (mri.py:11-163)."""

    def __init__(self, mask: Tensor | None = None, img_size: tuple | None = (320, 320), three_d: bool = False,
                 device="cpu", **kwargs):
        super().__init__(device=device, **kwargs)
        self.three_d = three_d
        self.img_size = img_size
        if mask is None:
            mask = torch.ones(*img_size, device=device)
        m = self.check_mask(mask, three_d=three_d)
        self.register_buffer("mask", m if m.is_floating_point() else m.to(torch.float32))
        self.img_size = self.mask.shape[1:]
        self._mcache = _MaskCache()
        self._aty_key = None
        self._aty = None
        self.to(device)

    # ---- helpers -------------------------------------------------------------------------------
    def _spec(self) -> ops.MaskSpec:
        return self._mcache.get(self.mask, self.three_d)

    def _dims(self) -> tuple:
        """(H, W), or (D, H, W) for three_d"""
        return tuple(int(s) for s in self.mask.shape[(-3 if self.three_d else -2):])

    def _op(self, t: Tensor, fwd: bool, inv: bool, gmode: int, **kw) -> Tensor:
        """one fused call of the 2-D (three_d: 3-D) spectral entry with this operator's mask"""
        fn = ops.spectral3d if self.three_d else ops.spectral
        return fn(t, *self._dims(), fwd=fwd, inv=inv, gmode=gmode, mask=self._spec(), **kw)

    def _check(self, t: Tensor):
        dims = self._dims()
        if t.dim() != 2 + len(dims) or t.shape[1] != 2 or tuple(t.shape[2:]) != dims:
            raise ValueError(f"expected a (B,2,{','.join(map(str, dims))}) tensor, got {tuple(t.shape)}")
        mb = self.mask.shape[0]
        if mb != 1 and mb != t.shape[0]:
            raise ValueError(f"mask batch {mb} does not match input batch {t.shape[0]}")

    def V_adjoint(self, x: Tensor) -> Tensor:
        return self.im_to_kspace(x, three_d=self.three_d)

    def V(self, x: Tensor, **kwargs) -> Tensor:
        return self.kspace_to_im(x, three_d=self.three_d)

    def U(self, x):
        return x

    def U_adjoint(self, x, **kwargs):
        return x

    # ---- fused operator bodies ---------------------------------------------------------------
    def _A(self, x, gmode=_ffi.G_MASK):
        return self._op(x, True, False, gmode)

    def _At(self, y, gmode=_ffi.G_MASK):
        return self._op(y, False, True, gmode)

    def A(self, x: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        self._check(x)
        return linear_apply(x, self._A, self._At)

    def A_adjoint(self, y: Tensor, mask: Tensor = None, mag: bool = False, crop: bool = False, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        self._check(y)
        x = linear_apply(y, self._At, self._A)
        if mag:
            x = self.rss(x, multicoil=False)
        if crop:
            x = self.crop(x, crop=crop)
        return x

    def A_adjoint_A(self, x: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        self._check(x)
        f = lambda t: self._op(t, True, True, _ffi.G_SQ)
        return linear_apply(x, f, f)

    def A_A_adjoint(self, y: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        self._check(y)
        f = lambda t: self._op(t, False, False, _ffi.G_SQ)
        return linear_apply(y, f, f)

    def A_dagger(self, y: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        self._check(y)
        if torch.is_grad_enabled() and y.requires_grad:
            return super().A_dagger(y)
        return self._At(y, gmode=_ffi.G_PINV)

    def _cached_At(self, y: Tensor) -> Tensor:
        """A^T y for a constant y (the reference recomputes it every iteration, data_fidelity.py:335-336)"""
        if not cache_hit(self._aty_key, y, self.mask):
            self._aty = self._At(y)
            self._aty_key = TensorKey(y, self.mask)
        return self._aty

    def prox_l2(self, z: Tensor, y: Tensor, gamma, **kwargs) -> Tensor:
        r"""argmin_x gamma/2 ||Ax-y||^2 + 1/2 ||x-z||^2 = V((V^T(A^T y + z/gamma)) / (s^2 + 1/gamma)) (forward.py:1212-1234)"""
        needs_grad = torch.is_grad_enabled() and (z.requires_grad or y.requires_grad or
                                                  (isinstance(gamma, Tensor) and gamma.requires_grad))
        if needs_grad:
            return super().prox_l2(z, y, gamma, **kwargs)
        self._check(z)
        aty = self._cached_At(y)
        if isinstance(gamma, Tensor) and gamma.numel() > 1:
            g = gamma.reshape(-1).to(device=z.device, dtype=torch.float32)
            if g.numel() != z.shape[0]:
                raise ValueError("per-sample gamma must have one entry per batch element")
            zg = z / g.reshape(-1, *([1] * (z.dim() - 1)))
            return self._op(aty, True, True, _ffi.G_INV_SQ_PLUS_C, p1=zg, a1=1.0, c_batch=(1.0 / g).contiguous())
        g = float(gamma)
        return self._op(aty, True, True, _ffi.G_INV_SQ_PLUS_C, p1=z, a1=1.0 / g, c=1.0 / g)

    def normal_step(self, x: Tensor, aty: Tensor, gamma: float) -> Tensor:
        r"""fused gradient step of the L2 data term: x - gamma * (A^T A x - A^T y)
        (optim_iterators/pgd.py:137-139 with data_fidelity.py:335-336) in one launch for line masks"""
        self._check(x)
        return self._op(x, True, True, _ffi.G_SQ, e0=-gamma, q0=x, e1=1.0, q1=aty, e2=gamma)

    def noise(self, x, **kwargs):
        return self.U(self.noise_model(x, **kwargs) * self.mask)

    def update_parameters(self, mask: Tensor = None, check_mask: bool = True, **kwargs):
        if mask is not None:
            mask = self.check_mask(mask=mask, three_d=getattr(self, "three_d", False)) if check_mask else mask
        super().update_parameters(mask=mask, **kwargs)


class TimeMixin:
    """time <-> batch folding helpers (deepinv/utils/mixins.py:19-115)"""

    @staticmethod
    def flatten(x: Tensor) -> Tensor:
        B, C, T, H, W = x.shape
        return x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)

    @staticmethod
    def unflatten(x: Tensor, batch_size: int = 1, frames: int | None = None) -> Tensor:
        BT, C, H, W = x.shape
        T = frames if frames is not None else BT // batch_size  # `frames` makes the empty batch well defined
        return x.reshape(batch_size, T, C, H, W).permute(0, 2, 1, 3, 4)

    @staticmethod
    def flatten_C(x: Tensor) -> Tensor:
        return x.reshape(x.shape[0], x.shape[1] * x.shape[2], x.shape[3], x.shape[4])

    @staticmethod
    def average(x: Tensor, mask: Tensor = None, dim: int = 2) -> Tensor:
        _x = x.sum(dim)
        out = torch.zeros_like(_x)
        m = (mask if mask is not None else (x != 0)).sum(dim)
        out[m != 0] = _x[m != 0] / m[m != 0]
        return out

    @staticmethod
    def repeat(x: Tensor, target: Tensor, dim: int = 2) -> Tensor:
        return x.unsqueeze(dim=dim).expand_as(target)


class DynamicMRI(MRI, TimeMixin):
    r"""Single-coil dynamic (2-D + t) MRI  y_t = M_t F x_t  on (B,2,T,H,W) tensors (mri.py:499-598).

    Time frames are independent 2-D problems, so the operator is the static one on the time-folded batch: an internal
    `MRI` whose mask is the (B*T,2,H,W) folding of the 5-D `mask` buffer runs the same fused spectral kernels
    (A, A^T, A^T A, prox_l2, data step); only the fold / unfold permutes are extra.  Mask shapes accepted: (H,W), (T,H,W),
    (C,T,H,W), (B,C,T,H,W) like the reference."""

    def __init__(self, mask: Tensor | None = None, img_size: tuple | None = (320, 320), three_d: bool = False,
                 device="cpu", **kwargs):
        super().__init__(mask=mask, img_size=img_size, three_d=three_d, device=device, **kwargs)
        self._flat = None
        self._flat_key = None

    def check_mask(self, mask: Tensor = None, **kwargs) -> Tensor:
        if isinstance(mask, np.ndarray):
            mask = torch.from_numpy(mask)
        while mask is not None and len(mask.shape) < 5:  # to B,C,T,H,W
            mask = mask.unsqueeze(0)
        return MRIMixin.check_mask(mask, three_d=True)  # only pads C to 2 at this point

    def _static(self, batch: int) -> MRI:
        """the static operator on the time-folded batch (rebuilt when the mask buffer or the batch size changes)"""
        m = self.mask
        if not cache_hit(self._flat_key, m, extra=(batch,)):
            mb = m if (m.shape[0] == batch or batch == 1) else m.expand(batch, *m.shape[1:])
            self._flat = MRI(mask=self.flatten(mb).contiguous(), img_size=(2, *m.shape[-2:]), device=m.device)
            self._flat_key = TensorKey(m, extra=(batch,))
        return self._flat

    def _check(self, t: Tensor):
        Bm, _, T, H, W = self.mask.shape
        if t.dim() != 5 or t.shape[1] != 2 or tuple(t.shape[2:]) != (T, H, W):
            raise ValueError(f"expected a (B,2,{T},{H},{W}) tensor, got {tuple(t.shape)}")
        if Bm != 1 and Bm != t.shape[0]:
            raise ValueError(f"mask batch {Bm} does not match input batch {t.shape[0]}")

    def _fold(self, name: str, t: Tensor, *extra, **kw) -> Tensor:
        self._check(t)
        B = t.shape[0]
        out = getattr(self._static(B), name)(self.flatten(t), *extra, **kw)
        return self.unflatten(out, batch_size=B, frames=t.shape[2])

    def A(self, x: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        return self._fold("A", x)

    def A_adjoint(self, y: Tensor, mask: Tensor = None, mag: bool = False, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        return self._fold("A_adjoint", y, mag=mag)

    def A_dagger(self, y: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        return self.A_adjoint(y, mask=mask, **kwargs)

    def A_adjoint_A(self, x: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        return self._fold("A_adjoint_A", x)

    def A_A_adjoint(self, y: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        return self._fold("A_A_adjoint", y)

    def V_adjoint(self, x: Tensor) -> Tensor:
        return self._fold("V_adjoint", x)

    def V(self, x: Tensor, **kwargs) -> Tensor:
        return self._fold("V", x)

    def prox_l2(self, z: Tensor, y: Tensor, gamma, **kwargs) -> Tensor:
        self._check(z)
        B, T = z.shape[0], z.shape[2]
        if isinstance(gamma, Tensor) and gamma.numel() > 1:
            gamma = gamma.reshape(B, 1).expand(B, T).reshape(-1)
        return self.unflatten(self._static(B).prox_l2(self.flatten(z), self.flatten(y), gamma, **kwargs), batch_size=B, frames=T)

    def normal_step(self, x: Tensor, aty: Tensor, gamma: float) -> Tensor:
        self._check(x)
        B = x.shape[0]
        return self.unflatten(self._static(B).normal_step(self.flatten(x), self.flatten(aty), gamma), batch_size=B,
                              frames=x.shape[2])

    def noise(self, x, **kwargs):
        return self.noise_model(x, **kwargs) * self.mask

    def update_parameters(self, mask: Tensor = None, check_mask: bool = True, **kwargs):
        if mask is not None and check_mask:
            mask = self.check_mask(mask=mask)
        DecomposablePhysics.update_parameters(self, mask=mask, **kwargs)

    def to_static(self, mask: Tensor | None = None, device="cpu") -> MRI:
        """drop the time dimension: union of the per-frame masks (mri.py:583-598)"""
        return MRI(mask=torch.clip(self.mask.sum(2), 0.0, 1.0) if mask is None else mask, img_size=self.img_size,
                   device=device)


class SequentialMRI(DynamicMRI):
    r"""Sequential sampling of ONE static image: y_t = M_t F x, x (B,2,H,W), y (B,2,T,H,W) (mri.py:601-695).

    F x does not depend on t, so `A` runs ONE 2-D transform (the reference repeats x T times and transforms every copy)
    and then applies the T frame masks; the default adjoint averages the frames in k-space and runs one fused
    mask + inverse-transform launch of the static operator."""

    def A(self, x: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, **kwargs)
        if torch.is_grad_enabled() and x.requires_grad:
            return DynamicMRI.A(self, self.repeat(x, self.mask if x.shape[0] == self.mask.shape[0] else
                                                  self.mask.expand(x.shape[0], *self.mask.shape[1:])))
        k = MRIMixin.im_to_kspace(self, x)
        return k.unsqueeze(2) * self.mask

    def A_adjoint(self, y: Tensor, mask: Tensor = None, keep_time_dim: bool = False, **kwargs) -> Tensor:
        if keep_time_dim:
            return super().A_adjoint(y, mask, **kwargs)
        mask = self.check_mask(mask) if mask is not None else self.mask
        return self.to_static(device=y.device).A_adjoint(self.average(y, mask), mask=self.average(mask), **kwargs)

    def A_dagger(self, y: Tensor, mask: Tensor = None, **kwargs) -> Tensor:
        return self.A_adjoint(y, mask=mask, **kwargs)


class MultiCoilMRI(MRIMixin, LinearPhysics):
    r"""y_n = M F (S_n x) (mri.py:166-497); coil multiply, FFT and mask are one fused two-pass launch,
    the adjoint's coil combination is fused after the inverse transform.  With three_d=True x is (B,2,D,H,W), y
    (B,2,N,D,H,W) and every method runs on `dinvk_spectral3d` for any N >= 1; `A_adjoint(rss=True)` returns the RSS volume
    (B,1,D,H,W), where the reference raises ValueError (its `rss` call omits three_d)."""

    def __init__(self, mask: Tensor | None = None, coil_maps: Tensor | int | None = None,
                 img_size: tuple | None = (320, 320), three_d: bool = False, device="cpu", **kwargs):
        super().__init__(device=device, **kwargs)
        self.img_size = img_size
        self.three_d = three_d
        if mask is None:
            mask = torch.ones(*img_size, device=device)
        if coil_maps is None:
            coil_maps = torch.ones(self.img_size[-3:] if three_d else self.img_size[-2:], dtype=torch.complex64, device=device)
        elif isinstance(coil_maps, int):
            raise ImportError("sigpy is required to simulate coil maps; pass a complex64 tensor of maps instead")
        self.register_buffer("mask", self.check_mask(mask, three_d=three_d))
        self.register_buffer("coil_maps", self.check_coil_maps(coil_maps, three_d=three_d))
        self._mcache = _MaskCache()
        self.to(device)

    @staticmethod
    def check_coil_maps(coil_maps: Tensor, three_d: bool = False) -> Tensor:
        while len(coil_maps.shape) < (4 if not three_d else 5):
            coil_maps = coil_maps.unsqueeze(0)
        if not coil_maps.is_complex():
            raise ValueError("coil_maps should be of torch complex dtype.")
        return coil_maps

    def _spec(self):
        m = self.mask
        return self._mcache.get(m if m.dtype == torch.float32 else m.float(), self.three_d)

    def _maps(self) -> Tensor:
        cm = self.coil_maps
        return cm if cm.dtype == torch.complex64 else cm.to(torch.complex64)

    def _check3d(self, t: Tensor, coil_dim: bool):
        """shapes the 3-D kernels index by: volumes of the mask's (D,H,W) and mask / maps batches of 1 or B"""
        dims = tuple(self.mask.shape[-3:])
        ok = t.dim() == 5 + coil_dim and tuple(t.shape[-3:]) == dims and tuple(self.coil_maps.shape[-3:]) == dims
        if not ok or (coil_dim and t.shape[2] != self.coil_maps.shape[1]):
            raise ValueError(f"expected {'(B,2,N,D,H,W)' if coil_dim else '(B,2,D,H,W)'} with (D,H,W) = {dims} and "
                             f"N = {self.coil_maps.shape[1]} coils, got {tuple(t.shape)}")
        if self.mask.shape[0] not in (1, t.shape[0]):
            raise ValueError(f"mask batch {self.mask.shape[0]} does not match input batch {t.shape[0]}")

    def _A_general(self, x):
        H, W = x.shape[-2:]
        cm = self._maps()
        N = cm.shape[1]
        if self.three_d:
            self._check3d(x, False)
            return ops.spectral3d(x, *x.shape[-3:], fwd=True, inv=False, gmode=_ffi.G_MASK, mask=self._spec(), ncoil=N,
                                  coil_mode=1, coil_maps=cm)
        if N > 1:
            return ops.spectral(x, H, W, fwd=True, inv=False, gmode=_ffi.G_MASK, mask=self._spec(), ncoil=N,
                                coil_mode=1, coil_maps=cm)
        # single coil: multiply by the map with torch (tiny), then the plain kernel
        xc = self.from_torch_complex(cm[:, 0] * self.to_torch_complex(x)).contiguous()
        return ops.spectral(xc, H, W, fwd=True, inv=False, gmode=_ffi.G_MASK, mask=self._spec()).unsqueeze(2)

    def _At_general(self, y, rss=False):
        H, W = y.shape[-2:]
        cm = self._maps()
        N = y.shape[2]
        if self.three_d:
            self._check3d(y, True)
            return ops.spectral3d(y, *y.shape[-3:], fwd=False, inv=True, gmode=_ffi.G_MASK, mask=self._spec(), ncoil=N,
                                  coil_mode=3 if rss else 2, coil_maps=cm)
        if N > 1:
            return ops.spectral(y, H, W, fwd=False, inv=True, gmode=_ffi.G_MASK, mask=self._spec(), ncoil=N,
                                coil_mode=3 if rss else 2, coil_maps=cm)
        v = ops.spectral(y[:, :, 0].contiguous(), H, W, fwd=False, inv=True, gmode=_ffi.G_MASK, mask=self._spec())
        if rss:
            return self.rss(v.unsqueeze(2), multicoil=True)
        return self.from_torch_complex(torch.conj(cm[:, 0]) * self.to_torch_complex(v)).contiguous()

    def A(self, x: Tensor, mask: Tensor = None, coil_maps: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, coil_maps=coil_maps, **kwargs)
        self._check_coils(x.shape[0])
        return linear_apply(x, self._A_general, self._At_general)

    def A_adjoint(self, y: Tensor, mask: Tensor = None, coil_maps: Tensor = None, rss: bool = False,
                  crop: bool = False, **kwargs) -> Tensor:
        if y.shape[1] != 2:
            raise ValueError("y must be of shape (B,2,N,...,H,W)")
        self.update_parameters(mask=mask, coil_maps=coil_maps, **kwargs)
        self._check_coils(y.shape[0])
        if rss:
            x = self._At_general(y, rss=True)
        else:
            x = linear_apply(y, self._At_general, self._A_general)
        return self.crop(x, crop=crop)

    def _check_coils(self, batch):
        cb = self.coil_maps.shape[0]
        if cb != 1 and cb != batch:
            raise ValueError(f"coil_maps batch {cb} does not match input batch {batch}")

    def noise(self, x, **kwargs) -> Tensor:
        return self.mask[:, :, None] * self.noise_model(x, **kwargs)

    def A_dagger(self, y: Tensor, mask: Tensor = None, coil_maps: Tensor = None, **kwargs) -> Tensor:
        self.update_parameters(mask=mask, coil_maps=coil_maps)
        return super().A_dagger(y, **kwargs)

    def update_parameters(self, mask: Tensor = None, coil_maps: Tensor = None, check_mask: bool = True,
                          check_coil_maps: bool = True, **kwargs):
        if mask is not None:
            mask = self.check_mask(mask=mask, three_d=self.three_d) if check_mask else mask
        if coil_maps is not None:
            coil_maps = self.check_coil_maps(coil_maps, three_d=self.three_d) if check_coil_maps else coil_maps
        super().update_parameters(mask=mask, coil_maps=coil_maps, **kwargs)
        self.img_size = self.mask.shape[1:]
        if self.coil_maps is not None and self.coil_maps.shape[2:] != self.img_size[1:]:
            warn(f"After updating parameters, img_size {self.img_size} in MultiCoilMRI is incompatible with coil_maps "
                 f"shape {self.coil_maps.shape} in the spatial dims.")
