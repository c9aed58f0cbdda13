"""Thin torch-tensor front end of the C ABI (pointers + sizes go down, nothing else).

Every function here requires CUDA tensors and enqueues on torch's current stream.  Workspaces are
torch tensors cached per (device, size) so that calls are allocation-free after warm-up and can be
captured in CUDA graphs.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _ffi
from ._lib import DinvkError, check, get_lib

_ws_cache: dict[tuple, torch.Tensor] = {}
_ws_retired: list[torch.Tensor] = []  # outgrown workspaces stay alive: a captured CUDA graph may have their address baked in


def _require_cuda(*ts: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise DinvkError(
                "deepinv_b200 operators run on CUDA tensors only (no CPU fallback); got a tensor on " f"{t.device}"
            )
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise DinvkError(f"tensors on different devices: {dev} vs {t.device}")
    if dev is None:
        raise DinvkError("no tensor given")
    if dev.index is not None and dev.index != torch.cuda.current_device():
        # the library keys its tables by the CURRENT device and launches on the tensors' stream: make them agree (like a
        # torch op's device guard; stays switched, as `with torch.cuda.device(t.device)` around the caller would leave it)
        torch.cuda.set_device(dev)
    return dev


def _stream(dev: torch.device) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _p(t: Optional[torch.Tensor]) -> Optional[ctypes.c_void_p]:
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """fp32 + contiguous (inputs may be arbitrary views: the reference itself hands out transposed views)"""
    if t is None:
        return None
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def workspace(dev: torch.device, nbytes: int, tag: str = "") -> torch.Tensor:
    key = (dev, tag)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < nbytes:
        if ws is not None:
            _ws_retired.append(ws)  # never hand the old block back to the allocator (replaying an earlier graph would scribble on it)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        _ws_cache[key] = ws
    return ws


# --------------------------------------------------------------------------------------------
# spectral family
# --------------------------------------------------------------------------------------------
class MaskSpec:
    """Device-side description of a spectral multiplier (see `dinvk_spectral_args`)."""

    __slots__ = ("tensor", "sb", "sc", "sh", "complex")

    def __init__(self, tensor: torch.Tensor, sb: int, sc: int, sh: int, complex_: bool = False):
        self.tensor, self.sb, self.sc, self.sh, self.complex = tensor, sb, sc, sh, complex_


def mask_spec_from_real(mask: torch.Tensor, H: int, W: int, compress: bool = True) -> MaskSpec:
    """mask: (1|B, 2, H, W) fp32 as stored by the reference's MRI (`check_mask`, mixins.py:125-146).

    With compress=True a mask that is constant along H and identical on both planes (the reference's
    Cartesian line masks, physics/generator/mri.py:170-196) is stored as (B,1,1,W): the kernels then
    skip the H-direction transforms in A^T A / prox (see dinvk.h)."""
    m = _f32c(mask)
    assert m.dim() == 4 and m.shape[1] == 2 and m.shape[2] == H and m.shape[3] == W, f"mask shape {tuple(m.shape)}"
    B = m.shape[0]
    if compress and H > 1:
        row = m[:, :1, :1, :]
        if bool((m == row).all()):
            mc = row.contiguous()
            return MaskSpec(mc, W if B > 1 else 0, 0, 0)
    return MaskSpec(m, 2 * H * W if B > 1 else 0, H * W, W)


def spectral(
    p0: torch.Tensor,
    H: int,
    W: int,
    *,
    fwd: bool,
    inv: bool,
    centered: bool = True,
    gmode: int = _ffi.G_NONE,
    mask: Optional[MaskSpec] = None,
    a0: float = 1.0,
    p1: Optional[torch.Tensor] = None,
    a1: float = 0.0,
    c: float = 0.0,
    c_batch: Optional[torch.Tensor] = None,
    q0: Optional[torch.Tensor] = None,
    e1: float = 0.0,
    q1: Optional[torch.Tensor] = None,
    e2: float = 0.0,
    e0: float = 1.0,
    ncoil: int = 0,
    coil_mode: int = 0,
    coil_maps: Optional[torch.Tensor] = None,
    out: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """out = e0 * F^-1( g(mask) . F( a0*p0 + a1*p1 ) ) + e1*q0 + e2*q1 on planar (B,2,H,W) tensors."""
    dev = _require_cuda(p0, p1, q0, q1, c_batch, coil_maps, None if mask is None else mask.tensor)
    p0 = _f32c(p0)
    p1, q0, q1, c_batch = _f32c(p1), _f32c(q0), _f32c(q1), _f32c(c_batch)
    nc = ncoil if ncoil > 1 else 1
    if nc > 1 and coil_mode == 1:
        batch = p0.shape[0]
        nimg = batch * nc
        out_shape = (batch, 2, nc, H, W)
    elif nc > 1:
        batch = p0.shape[0]
        nimg = batch * nc
        out_shape = (batch, 2, H, W) if coil_mode == 2 else (batch, 1, H, W)
    else:
        nimg = p0.numel() // (2 * H * W)
        out_shape = tuple(p0.shape)
    if out is None:
        out = torch.empty(out_shape, dtype=torch.float32, device=dev)
    else:
        assert out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == tuple(out_shape)
    if out.numel() == 0:  # empty batch: nothing to launch (an empty tensor has a null data pointer)
        return out
    a = _ffi.SpectralArgs()
    a.B, a.H, a.W = nimg, H, W
    a.fwd, a.inv, a.centered, a.gmode = int(fwd), int(inv), int(centered), gmode
    a.p0, a.p1, a.a0, a.a1 = p0.data_ptr(), (p1.data_ptr() if p1 is not None else None), a0, a1
    if gmode != _ffi.G_NONE:
        if mask is None:
            raise DinvkError("spectral: gmode needs a mask")
        a.mask, a.mask_sb, a.mask_sc, a.mask_sh = mask.tensor.data_ptr(), mask.sb, mask.sc, mask.sh
    a.c = c
    a.c_batch = c_batch.data_ptr() if c_batch is not None else None
    a.q0, a.q1 = (q0.data_ptr() if q0 is not None else None), (q1.data_ptr() if q1 is not None else None)
    a.e0, a.e1, a.e2 = e0, e1, e2
    a.out = out.data_ptr()
    a.ncoil, a.coil_mode = (nc if nc > 1 else 0), coil_mode
    if coil_maps is not None:
        cm = coil_maps if coil_maps.is_contiguous() else coil_maps.contiguous()
        assert cm.dtype == torch.complex64
        a.coil_maps = cm.data_ptr()
        a.coil_sb = nc * H * W if cm.shape[0] > 1 else 0
    lib = get_lib()
    nbytes = lib.dinvk_spectral_workspace_bytes(nimg, H, W)
    ws = workspace(dev, nbytes, "spectral")
    check(lib.dinvk_spectral(ctypes.byref(a), _p(ws), ws.numel(), _stream(dev)))
    return out


def mask_spec3d(mask: torch.Tensor) -> MaskSpec:
    """mask: (1|B, 2, D, H, W) fp32 as stored by the reference's 3-D MRI operators (`check_mask(three_d=True)`)"""
    m = _f32c(mask)
    assert m.dim() == 5 and m.shape[1] == 2, f"mask shape {tuple(m.shape)}"
    D, H, W = m.shape[-3:]
    return MaskSpec(m, 2 * D * H * W if m.shape[0] > 1 else 0, D * H * W, W)


def spectral3d(
    p0: torch.Tensor,
    D: int,
    H: int,
    W: int,
    *,
    fwd: bool,
    inv: bool,
    centered: bool = True,
    gmode: int = _ffi.G_NONE,
    mask: Optional[MaskSpec] = None,
    a0: float = 1.0,
    p1: Optional[torch.Tensor] = None,
    a1: float = 0.0,
    c: float = 0.0,
    c_batch: Optional[torch.Tensor] = None,
    q0: Optional[torch.Tensor] = None,
    e1: float = 0.0,
    q1: Optional[torch.Tensor] = None,
    e2: float = 0.0,
    e0: float = 1.0,
    ncoil: int = 0,
    coil_mode: int = 0,
    coil_maps: Optional[torch.Tensor] = None,
    out: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """`spectral` on planar (B,2,...,D,H,W) volumes with the 3-D DFT over the last three dims.  coil_mode 1 / 2 / 3 work for any
    ncoil >= 1: x (batch,2,D,H,W) -> y (batch,2,ncoil,D,H,W), y -> x, y -> rss (batch,1,D,H,W); maps (1|batch, ncoil, D, H, W)
    complex64.  Without coils, the dims between the planes and the volume (e.g. the coils of a (B,2,N,D,H,W) k-space) are
    transformed volume by volume, with the mask of their sample."""
    dev = _require_cuda(p0, p1, q0, q1, c_batch, coil_maps, None if mask is None else mask.tensor)
    p0 = _f32c(p0)
    p1, q0, q1, c_batch = _f32c(p1), _f32c(q0), _f32c(q1), _f32c(c_batch)
    vol = D * H * W
    if coil_mode:
        nc = max(int(ncoil), 1)
        batch = p0.shape[0]
        nimg = batch * nc
        out_shape = {1: (batch, 2, nc, D, H, W), 2: (batch, 2, D, H, W), 3: (batch, 1, D, H, W)}[coil_mode]
    else:  # (B,2,...,D,H,W): the dims between the planes and the volume are a stack of volumes per sample (ncoil of the ABI)
        if p0.dim() < 5 or p0.shape[1] != 2 or tuple(p0.shape[-3:]) != (D, H, W):
            raise ValueError(f"spectral3d: expected a planar (B,2,...,{D},{H},{W}) tensor, got {tuple(p0.shape)}")
        nc = 1
        for s in p0.shape[2:-3]:
            nc *= int(s)
        nimg = p0.shape[0] * nc
        out_shape = tuple(p0.shape)
    if out is None:
        out = torch.empty(out_shape, dtype=torch.float32, device=dev)
    else:
        assert out.is_contiguous() and out.dtype == torch.float32 and tuple(out.shape) == tuple(out_shape)
    if out.numel() == 0:  # empty batch: nothing to launch (an empty tensor has a null data pointer)
        return out
    a = _ffi.SpectralArgs()
    a.B, a.H, a.W = nimg, H, W
    a.fwd, a.inv, a.centered, a.gmode = int(fwd), int(inv), int(centered), gmode
    a.p0, a.p1, a.a0, a.a1 = p0.data_ptr(), (p1.data_ptr() if p1 is not None else None), a0, a1
    if gmode != _ffi.G_NONE:
        if mask is None:
            raise DinvkError("spectral3d: gmode needs a mask")
        a.mask, a.mask_sb, a.mask_sc, a.mask_sh = mask.tensor.data_ptr(), mask.sb, mask.sc, mask.sh
    a.c = c
    a.c_batch = c_batch.data_ptr() if c_batch is not None else None
    a.q0, a.q1 = (q0.data_ptr() if q0 is not None else None), (q1.data_ptr() if q1 is not None else None)
    a.e0, a.e1, a.e2 = e0, e1, e2
    a.out = out.data_ptr()
    a.ncoil, a.coil_mode = (nc if nc > 1 or coil_mode else 0), coil_mode
    if coil_maps is not None:
        cm = coil_maps if coil_maps.is_contiguous() else coil_maps.contiguous()
        assert cm.dtype == torch.complex64
        a.coil_maps = cm.data_ptr()
        a.coil_sb = nc * vol if cm.shape[0] > 1 else 0
    lib = get_lib()
    nbytes = lib.dinvk_spectral3d_workspace_bytes(nimg, D, H, W)
    ws = workspace(dev, nbytes, "spectral")
    check(lib.dinvk_spectral3d(ctypes.byref(a), D, _p(ws), ws.numel(), _stream(dev)))
    return out


def fft_prepare(n: int, centered: bool = True) -> None:
    check(get_lib().dinvk_fft_prepare(n, int(centered)))


# --------------------------------------------------------------------------------------------
# elementwise / reductions
# --------------------------------------------------------------------------------------------
def axpbypcz(x, a: float, y=None, b: float = 0.0, z=None, c: float = 0.0, out=None) -> torch.Tensor:
    dev = _require_cuda(x, y, z)
    x, y, z = _f32c(x), _f32c(y), _f32c(z)
    if out is None:
        out = torch.empty_like(x)
    if x.numel() == 0:
        return out
    check(get_lib().dinvk_axpbypcz(_p(out), _p(x), a, _p(y), b, _p(z), c, x.numel(), _stream(dev)))
    return out


def batched_dot(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """(B,) fp32: sum over all non-batch dims of x*y"""
    dev = _require_cuda(x, y)
    x, y = _f32c(x), _f32c(y)
    B = x.shape[0]
    n_per = x.numel() // max(B, 1)
    out = torch.empty(B, dtype=torch.float32, device=dev)
    if B == 0:
        return out
    if n_per == 0:
        return out.zero_()
    lib = get_lib()
    nb = lib.dinvk_batched_dot_workspace_bytes(B, n_per)
    ws = workspace(dev, nb, "dot")
    check(lib.dinvk_batched_dot(_p(out), _p(x), _p(y), B, n_per, _p(ws), ws.numel(), _stream(dev)))
    return out


def batched_axpy(x: torch.Tensor, y: torch.Tensor, s: torch.Tensor, sa: float = 1.0, out=None) -> torch.Tensor:
    """out[b] = x[b] + sa * s[b] * y[b]"""
    dev = _require_cuda(x, y, s)
    x, y, s = _f32c(x), _f32c(y), _f32c(s)
    B = x.shape[0]
    if out is None:
        out = torch.empty_like(x)
    if x.numel() == 0:
        return out
    check(get_lib().dinvk_batched_axpy(_p(out), _p(x), _p(y), _p(s), sa, B, x.numel() // max(B, 1), _stream(dev)))
    return out


def cg_scalars(mode: int, num, den, eps: float, bnorm2=None, tol2: float = 0.0, done_flag=None) -> torch.Tensor:
    dev = _require_cuda(num, den)
    out = torch.empty_like(num)
    if num.numel() == 0:
        return out
    check(get_lib().dinvk_cg_scalars(mode, _p(out), _p(num), _p(den), eps, _p(bnorm2), tol2, _p(done_flag), num.numel(),
                                     _stream(dev)))
    return out


def ddrm_update(x_bar, x_bar_prev, y_bar, mask, noise, sigma_t, sigma_prev, sigma_noise, eta, etab, c_sig, eps, init):
    dev = _require_cuda(y_bar, mask, noise, x_bar, x_bar_prev)
    out = torch.empty_like(y_bar)
    check(get_lib().dinvk_ddrm_update(_p(out), _p(x_bar), _p(x_bar_prev), _p(y_bar), _p(mask), _p(noise), y_bar.numel(),
                                      mask.numel(), sigma_t, sigma_prev, sigma_noise, eta, etab, c_sig, eps, int(init),
                                      _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# denoiser convolutions, fp32 path
# --------------------------------------------------------------------------------------------
def conv_f32(x, weight, *, kind: int = 0, bias=None, xadd=None, res=None, relu: bool = False) -> torch.Tensor:
    dev = _require_cuda(x, weight, bias, xadd, res)
    x, weight, bias, xadd, res = _f32c(x), _f32c(weight), _f32c(bias), _f32c(xadd), _f32c(res)
    B, Cin, H, W = x.shape
    if kind == 2:
        Cout = weight.shape[1]
        out = torch.empty(B, Cout, 2 * H, 2 * W, dtype=torch.float32, device=dev)
    elif kind == 1:
        Cout = weight.shape[0]
        out = torch.empty(B, Cout, H // 2, W // 2, dtype=torch.float32, device=dev)
    else:
        Cout = weight.shape[0]
        out = torch.empty(B, Cout, H, W, dtype=torch.float32, device=dev)
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_conv_f32(_p(x), _p(xadd), _p(weight), _p(bias), _p(res), _p(out), B, Cin, Cout, H, W, kind,
                                   int(relu), _stream(dev)))
    return out


def conv_f32_wgrad(x, xadd, gout, weight_shape, kind: int = 0, want_bias: bool = False):
    """weight (and bias) gradient of `conv_f32`: x [+ xadd] is the forward input, gout the gradient of the
    pre-residual output; returns (dweight, dbias | None)"""
    dev = _require_cuda(x, xadd, gout)
    x, xadd, gout = _f32c(x), _f32c(xadd), _f32c(gout)
    B, Cin, H, W = x.shape
    Cout = weight_shape[1] if kind == 2 else weight_shape[0]
    dw = torch.empty(tuple(weight_shape), dtype=torch.float32, device=dev)
    db = torch.empty(Cout, dtype=torch.float32, device=dev) if want_bias else None
    check(get_lib().dinvk_conv_f32_wgrad(_p(x), _p(xadd), _p(gout), _p(dw), _p(db), B, Cin, Cout, H, W, kind, _stream(dev)))
    return dw, db


def relu_bwd(gout, out) -> torch.Tensor:
    dev = _require_cuda(gout, out)
    gout, out = _f32c(gout), _f32c(out)
    gin = torch.empty_like(gout)
    check(get_lib().dinvk_relu_bwd(_p(gout), _p(out), _p(gin), gout.numel(), _stream(dev)))
    return gin


class _ConvF32Fn(torch.autograd.Function):
    """differentiable `conv_f32`: out = act(conv(x + xadd, w) + bias) + res.  Backward (first order) runs on the same
    library: ReLU mask, data gradient through the forward entry (3x3: transposed + flipped filter; the 2x2 strided conv
    and its transpose are each other's data gradient), weight / bias gradient through `dinvk_conv_f32_wgrad`."""

    @staticmethod
    def forward(ctx, x, xadd, weight, bias, res, kind, relu):
        if relu and res is not None:  # the ReLU mask is recovered from the output, which the residual would hide
            raise NotImplementedError("conv_f32 backward: ReLU together with a residual is not used by DRUNet / DnCNN")
        out = conv_f32(x, weight, kind=kind, bias=bias, xadd=xadd, res=res, relu=relu)
        ctx.kind, ctx.relu = kind, relu
        ctx.has = (xadd is not None, bias is not None, res is not None)
        ctx.save_for_backward(x, xadd, weight, out if relu else None)
        return out

    @staticmethod
    def backward(ctx, g):
        x, xadd, weight, out = ctx.saved_tensors
        kind = ctx.kind
        has_xadd, has_bias, has_res = ctx.has
        need = ctx.needs_input_grad
        g = _f32c(g)
        gp = relu_bwd(g, out) if ctx.relu else g
        dx = dw = db = None
        if need[0] or (has_xadd and need[1]):
            if kind == 0:
                wt = weight.detach().transpose(0, 1).flip(2, 3).contiguous()
                dx = conv_f32(gp, wt)
            else:
                dx = conv_f32(gp, weight.detach(), kind=2 if kind == 1 else 1)
        if need[2] or (has_bias and need[3]):
            dw, db = conv_f32_wgrad(x, xadd, gp, weight.shape, kind=kind, want_bias=has_bias and need[3])
        return (dx if need[0] else None, dx if (has_xadd and need[1]) else None, dw if need[2] else None,
                db if (has_bias and need[3]) else None, g if (has_res and need[4]) else None, None, None)


def conv_f32_ag(x, weight, *, kind: int = 0, bias=None, xadd=None, res=None, relu: bool = False) -> torch.Tensor:
    """`conv_f32` that records a backward when (and only when) a gradient is being tracked"""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, weight, bias, xadd, res)):
        return _ConvF32Fn.apply(x, xadd, weight, bias, res, kind, relu)
    return conv_f32(x, weight, kind=kind, bias=bias, xadd=xadd, res=res, relu=relu)


# --------------------------------------------------------------------------------------------
# Radon family (sinograms live in angle-major memory (B, C, A, P); see csrc/radon.cu)
# --------------------------------------------------------------------------------------------
def radon_fwd(x, P: int, cos_t, sin_t, circle: bool, scale: float) -> torch.Tensor:
    dev = _require_cuda(x, cos_t, sin_t)
    x = _f32c(x)
    B, C, W, _ = x.shape
    A = cos_t.shape[-1]
    sino = torch.empty(B, C, A, P, dtype=torch.float32, device=dev)
    if sino.numel() == 0:
        return sino
    check(get_lib().dinvk_radon_fwd(_p(x), _p(sino), B * C, W, P, A, int(circle), _p(cos_t), _p(sin_t), scale, _stream(dev)))
    return sino


def radon_adj(sino_am, W: int, cos_t, sin_t, circle: bool, scale: float, iradon: bool = False) -> torch.Tensor:
    """sino_am: (B, C, A, P) contiguous angle-major"""
    dev = _require_cuda(sino_am, cos_t, sin_t)
    sino_am = _f32c(sino_am)
    B, C, A, P = sino_am.shape
    x = torch.empty(B, C, W, W, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    fn = get_lib().dinvk_iradon_bp if iradon else get_lib().dinvk_radon_adj
    check(fn(_p(sino_am), _p(x), B * C, W, P, A, int(circle), _p(cos_t), _p(sin_t), scale, _stream(dev)))
    return x


def fanbeam(t, W: int, G: int, D: int, cos_t, sin_t, circle: bool, half_len: float, src: float, den: float, scale: float,
            adjoint: bool) -> torch.Tensor:
    """fan-beam projector: image (B,C,W,W) -> angle-major sinogram (B,C,A,D), or its exact transpose"""
    dev = _require_cuda(t, cos_t, sin_t)
    t = _f32c(t)
    B, C = t.shape[:2]
    A = cos_t.shape[-1]
    out = torch.empty((B, C, W, W) if adjoint else (B, C, A, D), dtype=torch.float32, device=dev)
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_fanbeam(_p(t), _p(out), B * C, W, G, D, A, int(circle), _p(cos_t), _p(sin_t), half_len, src, den,
                                  scale, int(adjoint), _stream(dev)))
    return out


def ramp_filter(sino_am) -> torch.Tensor:
    """ramp-filter every detector row of an angle-major sinogram (B, C, A, P)"""
    dev = _require_cuda(sino_am)
    sino_am = _f32c(sino_am)
    P = sino_am.shape[-1]
    rows = sino_am.numel() // max(P, 1)
    if sino_am.numel() == 0:
        return torch.empty_like(sino_am)
    if rows == 1:  # the kernel filters rows in pairs
        two = torch.cat([sino_am.reshape(1, P), torch.zeros(1, P, device=dev)], 0)
        return ramp_filter(two.reshape(1, 1, 2, P))[..., :1, :].reshape(sino_am.shape)
    out = torch.empty_like(sino_am)
    lib = get_lib()
    ws = workspace(dev, int(lib.dinvk_ramp_filter_workspace_bytes(rows, P)), "ramp")
    check(lib.dinvk_ramp_filter(_p(sino_am), _p(out), rows, P, _p(ws), ws.numel(), _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# MATLAB-bicubic resize (csrc/blur.cu: resize_fwd_kernel / resize_adj_kernel); tables from physics/imresize.py
# --------------------------------------------------------------------------------------------
def resize_fwd(x, th, tw) -> torch.Tensor:
    """(B,C,H,W) -> (B,C,th.n_out,tw.n_out): both 1-D passes of the banded resize in one launch"""
    dev = _require_cuda(x)
    x = _f32c(x)
    B, C, H, W = x.shape
    if (H, W) != (th.n_in, tw.n_in):
        raise ValueError(f"resize: tables for a {th.n_in}x{tw.n_in} image, got {H}x{W}")
    y = torch.empty(B, C, th.n_out, tw.n_out, dtype=torch.float32, device=dev)
    if y.numel() == 0:
        return y
    bh, wh = th.on(dev)[:2]
    bw, ww = tw.on(dev)[:2]
    check(get_lib().dinvk_resize_fwd(_p(x), _p(y), B * C, H, W, th.n_out, tw.n_out, _p(bh), _p(wh), th.k, _p(bw), _p(ww), tw.k,
                                     tw.scale, _stream(dev)))
    return y


def resize_adj(y, th, tw) -> torch.Tensor:
    """the transpose of resize_fwd: (B,C,th.n_out,tw.n_out) -> (B,C,th.n_in,tw.n_in)"""
    dev = _require_cuda(y)
    y = _f32c(y)
    B, C, Ho, Wo = y.shape
    if (Ho, Wo) != (th.n_out, tw.n_out):
        raise ValueError(f"resize: tables for a {th.n_out}x{tw.n_out} measurement, got {Ho}x{Wo}")
    x = torch.empty(B, C, th.n_in, tw.n_in, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    ph, oh, wh = th.on(dev)[2:]
    pw, ow, ww = tw.on(dev)[2:]
    check(get_lib().dinvk_resize_adj(_p(y), _p(x), B * C, th.n_in, tw.n_in, Ho, Wo, _p(ph), _p(oh), _p(wh), _p(pw), _p(ow), _p(ww),
                                     tw.k, tw.scale, _stream(dev)))
    return x


# --------------------------------------------------------------------------------------------
# Blur (direct convolution)
# --------------------------------------------------------------------------------------------
def blur_fwd(x, filt, padding: int) -> torch.Tensor:
    dev = _require_cuda(x, filt)
    x, filt = _f32c(x), _f32c(filt)
    B, C, H, W = x.shape
    FB, FC, h, w = filt.shape
    shape = (B, C, H - h + 1, W - w + 1) if padding == _ffi.PAD_VALID else (B, C, H, W)
    y = torch.empty(shape, dtype=torch.float32, device=dev)
    if y.numel() == 0:
        return y
    check(get_lib().dinvk_blur_fwd(_p(x), _p(filt), _p(y), B, C, H, W, FB, FC, h, w, padding, _stream(dev)))
    return y


def blur_adj(y, filt, padding: int, H: int, W: int) -> torch.Tensor:
    dev = _require_cuda(y, filt)
    y, filt = _f32c(y), _f32c(filt)
    B, C = y.shape[:2]
    FB, FC, h, w = filt.shape
    x = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    lib = get_lib()
    nb = lib.dinvk_blur_adj_workspace_bytes(B, C, H, W, h, w, padding)
    ws = workspace(dev, nb, "blur")
    check(lib.dinvk_blur_adj(_p(y), _p(filt), _p(x), B, C, H, W, FB, FC, h, w, padding, _p(ws), ws.numel(), _stream(dev)))
    return x


def blur3d_fwd(x, filt, padding: int) -> torch.Tensor:
    """the 3-D blur of (B,C,D,H,W) volumes by (FB,FC,d,h,w) filters (csrc/blur.cu: blur3d_corr_kernel)"""
    dev = _require_cuda(x, filt)
    x, filt = _f32c(x), _f32c(filt)
    B, C, D, H, W = x.shape
    FB, FC, d, h, w = filt.shape
    shape = (B, C, D - d + 1, H - h + 1, W - w + 1) if padding == _ffi.PAD_VALID else (B, C, D, H, W)
    if min(shape[2:]) < 1:  # a volume smaller than the filter: the library's argument check raises
        check(get_lib().dinvk_blur3d_fwd(_p(x), _p(filt), _p(x), B, C, D, H, W, FB, FC, d, h, w, padding, _stream(dev)))
    y = torch.empty(shape, dtype=torch.float32, device=dev)
    if y.numel() == 0:
        return y
    check(get_lib().dinvk_blur3d_fwd(_p(x), _p(filt), _p(y), B, C, D, H, W, FB, FC, d, h, w, padding, _stream(dev)))
    return y


def blur3d_adj(y, filt, padding: int, D: int, H: int, W: int) -> torch.Tensor:
    """the transpose of blur3d_fwd onto a (B,C,D,H,W) volume"""
    dev = _require_cuda(y, filt)
    y, filt = _f32c(y), _f32c(filt)
    B, C = y.shape[:2]
    FB, FC, d, h, w = filt.shape
    x = torch.empty(B, C, D, H, W, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    lib = get_lib()
    nb = lib.dinvk_blur3d_adj_workspace_bytes(B, C, D, H, W, d, h, w, padding)
    ws = workspace(dev, nb, "blur")
    check(lib.dinvk_blur3d_adj(_p(y), _p(filt), _p(x), B, C, D, H, W, FB, FC, d, h, w, padding, _p(ws), ws.numel(),
                               _stream(dev)))
    return x


def _svblur_shapes(mult, filt, B: int, C: int, H: int, W: int):
    MB, MC, K, Hm, Wm = mult.shape
    FB, FC, Kf, h, w = filt.shape
    if Kf != K or (Hm, Wm) != (H, W):
        raise ValueError(f"svblur: multipliers {tuple(mult.shape)} / filters {tuple(filt.shape)} do not match K terms on a "
                         f"({B}, {C}, {H}, {W}) image")
    return MB, MC, FB, FC, K, h, w


def svblur_fwd(x, mult, filt, padding: int) -> torch.Tensor:
    """y = sum_k filt[:, :, k] * (mult[:, :, k] . x): x (B,C,H,W), mult (MB,MC,K,H,W), filt (FB,FC,K,h,w)"""
    dev = _require_cuda(x, mult, filt)
    x, mult, filt = _f32c(x), _f32c(mult), _f32c(filt)
    B, C, H, W = x.shape
    MB, MC, FB, FC, K, h, w = _svblur_shapes(mult, filt, B, C, H, W)
    shape = (B, C, H - h + 1, W - w + 1) if padding == _ffi.PAD_VALID else (B, C, H, W)
    y = torch.empty(shape, dtype=torch.float32, device=dev)
    if y.numel() == 0:
        return y
    check(get_lib().dinvk_svblur_fwd(_p(x), _p(mult), _p(filt), _p(y), B, C, H, W, MB, MC, FB, FC, K, h, w, padding, _stream(dev)))
    return y


def svblur_adj(y, mult, filt, padding: int, H: int, W: int) -> torch.Tensor:
    """the transpose of svblur_fwd onto a (B,C,H,W) image"""
    dev = _require_cuda(y, mult, filt)
    y, mult, filt = _f32c(y), _f32c(mult), _f32c(filt)
    B, C = y.shape[:2]
    MB, MC, FB, FC, K, h, w = _svblur_shapes(mult, filt, B, C, H, W)
    x = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    lib = get_lib()
    nb = lib.dinvk_svblur_adj_workspace_bytes(B, C, H, W, h, w, padding)
    ws = workspace(dev, nb, "svblur")
    check(lib.dinvk_svblur_adj(_p(y), _p(mult), _p(filt), _p(x), B, C, H, W, MB, MC, FB, FC, K, h, w, padding, _p(ws), ws.numel(),
                               _stream(dev)))
    return x


def _tiled_svblur_shapes(mult, filt):
    _, _, K, P1, P2 = mult.shape
    FB, FC, Kf, h, w = filt.shape
    if Kf != K:
        raise ValueError(f"tiled_svblur: {K} multipliers for {Kf} filters")
    return FB, FC, K, h, w, P1, P2


def tiled_svblur_fwd(x, mult, filt, stride) -> torch.Tensor:
    """y = sum_k Wt_k . (filt[:, :, k] *valid x): x (B,C,H,W), mult (1,1,K,P1,P2), filt (FB,FC,K,h,w), stride (s1, s2)"""
    dev = _require_cuda(x, mult, filt)
    x, mult, filt = _f32c(x), _f32c(mult), _f32c(filt)
    B, C, H, W = x.shape
    FB, FC, K, h, w, P1, P2 = _tiled_svblur_shapes(mult, filt)
    y = torch.empty(B, C, H - h + 1, W - w + 1, dtype=torch.float32, device=dev)
    if y.numel() == 0:
        return y
    check(get_lib().dinvk_tiled_svblur_fwd(_p(x), _p(mult), _p(filt), _p(y), B, C, H, W, FB, FC, K, h, w, P1, P2, *stride,
                                           _stream(dev)))
    return y


def tiled_svblur_adj(y, mult, filt, stride, H: int, W: int) -> torch.Tensor:
    """the transpose of tiled_svblur_fwd onto a (B,C,H,W) image"""
    dev = _require_cuda(y, mult, filt)
    y, mult, filt = _f32c(y), _f32c(mult), _f32c(filt)
    B, C = y.shape[:2]
    FB, FC, K, h, w, P1, P2 = _tiled_svblur_shapes(mult, filt)
    x = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return x
    check(get_lib().dinvk_tiled_svblur_adj(_p(y), _p(mult), _p(filt), _p(x), B, C, H, W, FB, FC, K, h, w, P1, P2, *stride,
                                           _stream(dev)))
    return x


# --------------------------------------------------------------------------------------------
# denoiser convolutions, bf16 tensor-core path (NHWC bf16 activations)
# --------------------------------------------------------------------------------------------
def nchw_to_nhwc_bf16(x, cpad: int, fill=None) -> torch.Tensor:
    """(B,C,H,W) fp32 -> (B,H,W,cpad) bf16; `fill` (float or (B,) tensor) goes to channel C (DRUNet's noise map)"""
    dev = _require_cuda(x)
    x = _f32c(x)
    B, C, H, W = x.shape
    out = torch.empty(B, H, W, cpad, dtype=torch.bfloat16, device=dev)
    fb = _f32c(fill) if isinstance(fill, torch.Tensor) else None
    fs = float(fill) if (fill is not None and fb is None) else 0.0
    check(get_lib().dinvk_nchw_f32_to_nhwc_bf16(_p(x), _p(out), B, C, H, W, cpad, fs, _p(fb), int(fill is not None), _stream(dev)))
    return out


def nhwc_bf16_to_nchw(x, C: int, add=None) -> torch.Tensor:
    dev = _require_cuda(x)
    B, H, W, cpad = x.shape
    out = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    check(get_lib().dinvk_nhwc_bf16_to_nchw_f32(_p(x), _p(_f32c(add)), _p(out), B, C, H, W, cpad, _stream(dev)))
    return out


def conv3x3_bf16(x, w2d, *, bias=None, res=None, res2=None, relu: bool = False) -> torch.Tensor:
    """x (B,H,W,Cin) bf16, w2d (Cout, 9*Cin) bf16 -> (B,H,W,Cout) bf16 = act(conv + bias) + res + res2"""
    dev = _require_cuda(x, w2d)
    B, H, W, Cin = x.shape
    Cout = w2d.shape[0]
    out = torch.empty(B, H, W, Cout, dtype=torch.bfloat16, device=dev)
    check(get_lib().dinvk_conv3x3_bf16(_p(x), _p(w2d), _p(bias), _p(res), _p(res2), _p(out), B, H, W, Cin, Cout, int(relu),
                                       _stream(dev)))
    return out


def conv3x3_head_bf16(x, w64, *, bias=None, fill=None, relu: bool = False) -> torch.Tensor:
    """network head: (B,C,H,W) fp32 NCHW (+ constant channel `fill`: float or (B,) tensor) -> (B,H,W,64) bf16"""
    dev = _require_cuda(x, w64)
    x = _f32c(x)
    B, C, H, W = x.shape
    out = torch.empty(B, H, W, 64, dtype=torch.bfloat16, device=dev)
    fill_t = _f32c(fill.reshape(-1)) if torch.is_tensor(fill) else None
    if fill_t is not None and fill_t.numel() == 1:
        fill_t = fill_t.expand(B).contiguous()
    check(get_lib().dinvk_conv3x3_head_bf16(_p(x), _p(w64), _p(bias), _p(out), B, C, H, W,
                                            float(fill) if (fill is not None and fill_t is None) else 0.0,
                                            _p(fill_t), int(fill is not None), int(relu), _stream(dev)))
    return out


def conv3x3_bf16_tail(x, w16, cout: int, *, bias=None, add=None) -> torch.Tensor:
    """network tail: (B,H,W,Cin) bf16 -> (B,cout,H,W) fp32 NCHW (+ bias + add)"""
    dev = _require_cuda(x, w16)
    B, H, W, Cin = x.shape
    out = torch.empty(B, cout, H, W, dtype=torch.float32, device=dev)
    check(get_lib().dinvk_conv3x3_bf16_tail(_p(x), _p(w16), _p(bias), _p(_f32c(add)), _p(out), B, H, W, Cin, cout, _stream(dev)))
    return out


def conv2x2_bf16(x, w2d, cout: int, *, up: bool, xadd=None) -> torch.Tensor:
    dev = _require_cuda(x, w2d)
    B, H, W, Cin = x.shape
    shape = (B, 2 * H, 2 * W, cout) if up else (B, H // 2, W // 2, cout)
    out = torch.empty(shape, dtype=torch.bfloat16, device=dev)
    fn = get_lib().dinvk_conv2x2_up_bf16 if up else get_lib().dinvk_conv2x2_down_bf16
    check(fn(_p(x), _p(xadd), _p(w2d), _p(out), B, H, W, Cin, cout, _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# denoiser convolutions, fp32-grade tensor-core path (split operands; activations (B,H,W,C/CH,2,CH):
#   fp32 words, CH = 16  -> fmt 0 (3 x TF32);   fp16 words, CH = 32 -> fmt 1 (3 x FP16, |v| < 65504))
# --------------------------------------------------------------------------------------------
def _fmt_of(t: torch.Tensor) -> int:
    return 1 if t.dtype == torch.float16 else 0


def _split_empty(B, H, W, C, fmt, dev):
    ch, dt = (32, torch.float16) if fmt == 1 else (16, torch.float32)
    return torch.empty(B, H, W, C // ch, 2, ch, dtype=dt, device=dev)


def conv_tc32(x, w, cout: int, *, kind: int = 0, bias=None, res=None, res2=None, relu: bool = False, window: int = 0,
              flag=None) -> torch.Tensor:
    """x split layout, w packed by models.tc_engine._pack_tc32 -> split output
    kind 0: 3x3 (same grid), 1: 2x2 stride 2 (H/2, W/2), 2: transposed 2x2 stride 2 (2H, 2W);
    out = act(conv + bias) + res + res2;  flag: int32 overflow flag of the network (fp16 format)"""
    dev = _require_cuda(x, w)
    fmt = _fmt_of(x)
    B, H, W, nblk = x.shape[:4]
    Cin = nblk * x.shape[-1]
    Ho, Wo = (H, W) if kind == 0 else ((H // 2, W // 2) if kind == 1 else (2 * H, 2 * W))
    out = _split_empty(B, Ho, Wo, cout, fmt, dev)
    check(get_lib().dinvk_conv_tc32(_p(x), _p(w), _p(bias), _p(res), _p(res2), _p(out), B, H, W, Cin, cout, kind, int(relu),
                                    int(window), fmt, _p(flag), _stream(dev)))
    return out


def conv_tc32_slab(x, w, cout: int, *, bias=None, res=None, res2=None, relu: bool = False, window: int = 0, flag=None) -> torch.Tensor:
    """3x3 convolution with halo reuse (the body layers); w packed by models.tc_engine._pack3x3_slab_tc32; window in channel blocks"""
    dev = _require_cuda(x, w)
    fmt = _fmt_of(x)
    B, H, W, nblk = x.shape[:4]
    out = _split_empty(B, H, W, cout, fmt, dev)
    check(get_lib().dinvk_conv_tc32_slab(_p(x), _p(w), _p(bias), _p(res), _p(res2), _p(out), B, H, W, nblk * x.shape[-1], cout, int(relu),
                                         int(window), fmt, _p(flag), _stream(dev)))
    return out


def conv_tc32_head(x, weight, *, bias=None, fill=None, relu: bool = False, fmt: int = 0, flag=None) -> torch.Tensor:
    """network head: (B,C,H,W) fp32 NCHW (+ constant channel `fill`) -> split layout; weight (Cout,C[+1],3,3) fp32"""
    dev = _require_cuda(x, weight)
    x = _f32c(x)
    B, C, H, W = x.shape
    cout = weight.shape[0]
    out = _split_empty(B, H, W, cout, fmt, dev)
    fill_t = _f32c(fill.reshape(-1)) if torch.is_tensor(fill) else None
    if fill_t is not None and fill_t.numel() == 1:
        fill_t = fill_t.expand(B).contiguous()
    check(get_lib().dinvk_conv_tc32_head(_p(x), _p(_f32c(weight)), _p(bias), _p(out), B, C, H, W, cout,
                                         float(fill) if (fill is not None and fill_t is None) else 0.0,
                                         _p(fill_t), int(fill is not None), int(relu), fmt, _p(flag), _stream(dev)))
    return out


def conv_tc32_tail(x, weight, *, bias=None, add=None, flag=None) -> torch.Tensor:
    """network tail: split layout -> (B,Cout,H,W) fp32 NCHW (+ bias + add); weight (Cout,Cin,3,3) fp32, Cout <= 4;
    NaN if the network's overflow flag is set"""
    dev = _require_cuda(x, weight)
    B, H, W, nblk = x.shape[:4]
    cout = weight.shape[0]
    out = torch.empty(B, cout, H, W, dtype=torch.float32, device=dev)
    check(get_lib().dinvk_conv_tc32_tail(_p(x), _p(_f32c(weight)), _p(bias), _p(_f32c(add)), _p(out), B, H, W, nblk * x.shape[-1], cout,
                                         _fmt_of(x), _p(flag), _stream(dev)))
    return out


def conv3d_f32(x, weight, *, kind: int = 0, bias=None, xadd=None, res=None, relu: bool = False) -> torch.Tensor:
    """3-D `conv_f32` on (B, C, D, H, W): kind 0: 3x3x3 pad 1, 1: 2x2x2 stride 2, 2: transposed 2x2x2 stride 2 (forward only)"""
    dev = _require_cuda(x, weight, bias, xadd, res)
    x, weight, bias, xadd, res = _f32c(x), _f32c(weight), _f32c(bias), _f32c(xadd), _f32c(res)
    B, Cin, D, H, W = x.shape
    Cout = weight.shape[1] if kind == 2 else weight.shape[0]
    scale = {0: (1, 1), 1: (1, 2), 2: (2, 1)}.get(kind, (1, 1))
    out = torch.empty(B, Cout, *(s * scale[0] // scale[1] for s in (D, H, W)), dtype=torch.float32, device=dev)
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_conv3d_f32(_p(x), _p(xadd), _p(weight), _p(bias), _p(res), _p(out), B, Cin, Cout, D, H, W, kind,
                                     int(relu), _stream(dev)))
    return out


def _split3d_empty(B, D, H, W, C, fmt, dev):
    ch, dt = (32, torch.float16) if fmt == 1 else (16, torch.float32)
    return torch.empty(B, D, H, W, C // ch, 2, ch, dtype=dt, device=dev)


def conv3d_tc32(x, w, cout: int, *, kind: int = 0, bias=None, res=None, res2=None, relu: bool = False, window: int = 0,
                flag=None) -> torch.Tensor:
    """x split volume (B, D, H, W, C/CH, 2, CH), w packed by models.tc_engine (27-tap, 2x2x2 down or up order) -> split output
    kind 0: 3x3x3 (same grid), 1: 2x2x2 stride 2, 2: transposed 2x2x2 stride 2;  out = act(conv + bias) + res + res2"""
    dev = _require_cuda(x, w)
    fmt = _fmt_of(x)
    B, D, H, W, nblk = x.shape[:5]
    Cin = nblk * x.shape[-1]
    f = {0: lambda s: s, 1: lambda s: s // 2, 2: lambda s: 2 * s}.get(kind, lambda s: s)
    out = _split3d_empty(B, f(D), f(H), f(W), cout, fmt, dev)
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_conv3d_tc32(_p(x), _p(w), _p(bias), _p(res), _p(res2), _p(out), B, D, H, W, Cin, cout, kind, int(relu),
                                      int(window), fmt, _p(flag), _stream(dev)))
    return out


def conv3d_tc32_head(x, weight, *, bias=None, fill=None, relu: bool = False, fmt: int = 0, flag=None) -> torch.Tensor:
    """3-D network head: (B,C,D,H,W) fp32 (+ constant channel `fill`) -> split volume; weight (Cout,C[+1],3,3,3) fp32"""
    dev = _require_cuda(x, weight)
    x = _f32c(x)
    B, C, D, H, W = x.shape
    cout = weight.shape[0]
    out = _split3d_empty(B, D, H, W, cout, fmt, dev)
    fill_t = _f32c(fill.reshape(-1)) if torch.is_tensor(fill) else None
    if fill_t is not None and fill_t.numel() == 1:
        fill_t = fill_t.expand(B).contiguous()
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_conv3d_tc32_head(_p(x), _p(_f32c(weight)), _p(bias), _p(out), B, C, D, H, W, cout,
                                           float(fill) if (fill is not None and fill_t is None) else 0.0,
                                           _p(fill_t), int(fill is not None), int(relu), fmt, _p(flag), _stream(dev)))
    return out


def conv3d_tc32_tail(x, weight, *, bias=None, add=None, flag=None) -> torch.Tensor:
    """3-D network tail: split volume -> (B,Cout,D,H,W) fp32 (+ bias + add); weight (Cout,Cin,3,3,3) fp32, Cout <= 4;
    NaN if the network's overflow flag is set"""
    dev = _require_cuda(x, weight)
    B, D, H, W, nblk = x.shape[:5]
    cout = weight.shape[0]
    out = torch.empty(B, cout, D, H, W, dtype=torch.float32, device=dev)
    if out.numel() == 0:
        return out
    check(get_lib().dinvk_conv3d_tc32_tail(_p(x), _p(_f32c(weight)), _p(bias), _p(_f32c(add)), _p(out), B, D, H, W, nblk * x.shape[-1],
                                           cout, _fmt_of(x), _p(flag), _stream(dev)))
    return out


def split16_to_nchw(x) -> torch.Tensor:
    dev = _require_cuda(x)
    B, H, W, nblk = x.shape[:4]
    C = nblk * x.shape[-1]
    out = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
    check(get_lib().dinvk_split16_to_nchw(_p(x), _p(out), B, C, H, W, _fmt_of(x), _stream(dev)))
    return out


def nchw_to_split16(x, fmt: int = 0) -> torch.Tensor:
    dev = _require_cuda(x)
    x = _f32c(x)
    B, C, H, W = x.shape
    out = _split_empty(B, H, W, C, fmt, dev)
    check(get_lib().dinvk_nchw_to_split16(_p(x), _p(out), B, C, H, W, fmt, _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# data input side
# --------------------------------------------------------------------------------------------
def interleaved_to_planar(z: torch.Tensor) -> torch.Tensor:
    """complex64 (B, ...) on the device -> planar fp32 (B, 2, ...) (the reference's from_torch_complex, mixins.py:148-156)"""
    dev = _require_cuda(z)
    if z.dtype != torch.complex64:
        z = z.to(torch.complex64)
    z = z.contiguous()
    B = z.shape[0]
    n = z[0].numel() if B else 0
    out = torch.empty((B, 2, *z.shape[1:]), dtype=torch.float32, device=dev)
    if B and n:
        check(get_lib().dinvk_interleaved_to_planar(_p(torch.view_as_real(z)), _p(out), B, n, _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# total variation (deepinv/models/tv.py, deepinv/optim/prior.py:485-611)
# --------------------------------------------------------------------------------------------
TV_CTRL_FIELDS = ("ticket", "it_done", "cur", "status", "replay_n", "conv_j1")
TV_RUNNING, TV_FINISHED, TV_REPLAY = 0, 1, 2


def tv_block(lib=None) -> tuple[int, int]:
    """(T, K): the tile edge and the iterations per launch libdinvk's TV prox was compiled with"""
    t, k = ctypes.c_int(0), ctypes.c_int(0)
    check((lib or get_lib()).dinvk_tv_block(ctypes.byref(t), ctypes.byref(k)))
    return t.value, k.value


def tv_drive(launch, read_ctrl, n_it_max: int, iters_per_launch: int, check_every: int) -> dict:
    """Host loop of the TV and TGV proxes.

    `launch(first, n)` enqueues n iteration blocks; `read_ctrl()` synchronises and returns the control block as a dict.
    Issues ceil(n_it_max / K) blocks, reading the control block every `check_every` launches and after the last one;
    a launch issued after convergence returns at entry.  If the break test passed inside a block, one more launch
    replays the iterations up to the break.  Returns the final control block plus the launch and synchronisation counts.
    """
    total = -(-int(n_it_max) // iters_per_launch)
    issued = syncs = 0
    ctrl = {"it_done": 0, "cur": 0, "status": TV_FINISHED, "conv_j1": 0}
    while issued < total:
        k = min(max(1, int(check_every)), total - issued)
        launch(issued == 0, k)
        issued += k
        ctrl = read_ctrl()
        syncs += 1
        if ctrl["status"] != TV_RUNNING:
            break
    if ctrl["status"] == TV_REPLAY:
        launch(False, 1)
        issued += 1
        ctrl = dict(ctrl, cur=ctrl["cur"] ^ 1, it_done=ctrl["it_done"] + ctrl["replay_n"], status=TV_FINISHED)
    ctrl.update(launches=issued, syncs=syncs)
    return ctrl


def read_ctrl(ws: torch.Tensor) -> dict:
    """the control block at the head of a TV / TGV prox workspace (a byte tensor), as a dict; synchronises"""
    return dict(zip(TV_CTRL_FIELDS, ws[:4 * len(TV_CTRL_FIELDS)].view(torch.int32).tolist()))


def _cp_prox(lib, stream, call, state, nb: int, K: int, n_it_max: int, check_every: int, stats: Optional[dict] = None,
             fill: Optional[float] = None):
    """Run one TV / TGV prox from `state`, a list of state tensors, and return (state after the solve, control block).

    `call(*a, *b, first, n, ws, nb, stream)` calls the library's entry point with the pointers of the ping-pong state
    buffers a and b.  a starts as a copy of `state`; b is scratch, left uninitialised unless `fill` is given.  A replay
    needs its launch's input intact, which is why the buffers alternate.  nb is the workspace size in bytes, K the
    iterations per launch.  Works on CPU tensors with a None stream.
    """
    a = [t.float().clone(memory_format=torch.contiguous_format) for t in state]
    b = [torch.empty_like(t) if fill is None else torch.full_like(t, fill) for t in a]
    ws = torch.empty(nb, dtype=torch.uint8, device=a[0].device)  # per call: the control block is the solve's state

    def launch(first, n):
        check(call(*map(_p, a), *map(_p, b), int(first), n, _p(ws), nb, stream), lib)

    ctrl = tv_drive(launch, lambda: read_ctrl(ws), n_it_max if a[0].numel() else 0, K, check_every)
    if stats is not None:
        stats.update(launches=ctrl["launches"], syncs=ctrl["syncs"], converged=bool(ctrl["conv_j1"]))
    return (b if ctrl["cur"] else a), ctrl


def tv_prox(y: torch.Tensor, lambd: torch.Tensor, x2: torch.Tensor, u2: torch.Tensor, l1: bool = False, tau: float = 0.01,
            rho: float = 1.99, n_it_max: int = 1000, crit: float = 1e-5, check_every: int = 16, stats: Optional[dict] = None):
    """TVDenoiser / TVL1Denoiser iterations from the state (x2 (B,C,H,W), u2 (B,C,H,W,2)); lambd (B,) on the device.

    Returns (x2, u2, iterations) with the iteration count as a 0-d int32 device tensor.  `stats`, if given, receives the
    launch and host-synchronisation counts of this call.
    """
    dev = _require_cuda(y, lambd, x2, u2)
    if y.dim() != 4:
        raise NotImplementedError(f"the TV prox is 2-D only: expected (B, C, H, W), got {tuple(y.shape)}")
    y, lambd = _f32c(y), _f32c(lambd)
    B, C, H, W = y.shape
    if lambd.numel() != B:
        raise DinvkError(f"lambd must hold one value per sample: {lambd.numel()} values for a batch of {B}")
    lib = get_lib()
    (x, u), ctrl = _cp_prox(
        lib, _stream(dev),
        lambda xa, ua, xb, ub, *run: lib.dinvk_tv_prox(_p(y), xa, ua, xb, ub, _p(lambd), B, C, H, W, int(n_it_max), float(crit),
                                                       float(tau), float(rho), int(l1), *run),
        [x2, u2], lib.dinvk_tv_prox_workspace_bytes(B, C, H, W), tv_block(lib)[1], n_it_max, check_every, stats)
    return x, u, torch.full((), ctrl["it_done"], dtype=torch.int32, device=dev)


def _tv_shape(x: torch.Tensor, what: str) -> None:
    if x.dim() != 4:
        raise NotImplementedError(f"{what} is 2-D only: expected a (B, C, H, W) tensor, got {tuple(x.shape)}")


def tv_nabla(x: torch.Tensor) -> torch.Tensor:
    """finite differences (B,C,H,W) -> (B,C,H,W,2) (tv.py:153-181)"""
    dev = _require_cuda(x)
    _tv_shape(x, "nabla")
    x = _f32c(x)
    out = torch.empty((*x.shape, 2), dtype=torch.float32, device=dev)
    if x.numel():
        check(get_lib().dinvk_tv_stencil(0, _p(x), _p(out), *x.shape, _stream(dev)))
    return out


def tv_nabla_adjoint(g: torch.Tensor) -> torch.Tensor:
    """adjoint of the finite differences (B,C,H,W,2) -> (B,C,H,W) (tv.py:183-218)"""
    dev = _require_cuda(g)
    if g.dim() != 5 or g.shape[-1] != 2:
        raise NotImplementedError(f"nabla_adjoint is 2-D only: expected a (B, C, H, W, 2) tensor, got {tuple(g.shape)}")
    g = _f32c(g)
    out = torch.empty(g.shape[:-1], dtype=torch.float32, device=dev)
    if g.numel():
        check(get_lib().dinvk_tv_stencil(1, _p(g), _p(out), *g.shape[:-1], _stream(dev)))
    return out


def tv_grad(x: torch.Tensor) -> torch.Tensor:
    """TV subgradient nabla_adjoint(Dx / |Dx|), 0 where |Dx| = 0 (prior.py:544-572)"""
    dev = _require_cuda(x)
    _tv_shape(x, "TVPrior.grad")
    x = _f32c(x)
    out = torch.empty_like(x)
    if x.numel():
        check(get_lib().dinvk_tv_stencil(2, _p(x), _p(out), *x.shape, _stream(dev)))
    return out


def tv_fn(x: torch.Tensor, l1: bool = False) -> torch.Tensor:
    """(B,) TV value: sum of |Dx| with the 2-norm (TVPrior.fn) or 1-norm (TVL1Prior.fn) over the differences"""
    dev = _require_cuda(x)
    _tv_shape(x, "TVPrior.fn")
    x = _f32c(x)
    B, C, H, W = x.shape
    out = torch.zeros(B, dtype=torch.float32, device=dev)
    if x.numel() == 0:
        return out
    lib = get_lib()
    nb = lib.dinvk_tv_fn_workspace_bytes(B, C, H, W)
    ws = workspace(dev, nb, "tv_fn")
    check(lib.dinvk_tv_fn(_p(out), _p(x), int(l1), B, C, H, W, _p(ws), ws.numel(), _stream(dev)))
    return out


# --------------------------------------------------------------------------------------------
# total generalized variation (deepinv/models/tgv.py)
# --------------------------------------------------------------------------------------------
def tgv_block(lib=None) -> tuple[int, int]:
    """(T, K): the tile edge and the iterations per launch libdinvk's TGV prox was compiled with"""
    t, k = ctypes.c_int(0), ctypes.c_int(0)
    check((lib or get_lib()).dinvk_tgv_block(ctypes.byref(t), ctypes.byref(k)))
    return t.value, k.value


def tgv_prox(y: torch.Tensor, tl1: torch.Tensor, l2: torch.Tensor, x2: torch.Tensor, r2: torch.Tensor, u2: torch.Tensor,
             tau: float = 0.01, rho: float = 1.99, n_it_max: int = 1000, crit: float = 1e-5, check_every: int = 16,
             stats: Optional[dict] = None):
    """TGVDenoiser iterations from the state (x2 (B,C,H,W), r2 (B,C,H,W,2), u2 (B,C,H,W,4)); tl1 = tau * lambda1 and
    l2 = lambda2, (B,) on the device.

    Returns (x2, r2, u2, iterations) with the iteration count as a 0-d int32 device tensor.  `stats`, if given, receives
    the launch and host-synchronisation counts of this call.  Driven by `tv_drive` with the TV prox's control block.
    """
    dev = _require_cuda(y, tl1, l2, x2, r2, u2)
    if y.dim() != 4:
        raise NotImplementedError(f"the TGV prox is 2-D only: expected (B, C, H, W), got {tuple(y.shape)}")
    y, tl1, l2 = _f32c(y), _f32c(tl1), _f32c(l2)
    B, C, H, W = y.shape
    if tl1.numel() != B or l2.numel() != B:
        raise DinvkError(f"tl1 and l2 must hold one value per sample: {tl1.numel()}, {l2.numel()} values for a batch of {B}")
    if r2.shape != (B, C, H, W, 2) or u2.shape != (B, C, H, W, 4) or x2.shape != y.shape:
        raise DinvkError(f"TGV state shapes {tuple(x2.shape)}, {tuple(r2.shape)}, {tuple(u2.shape)} do not match y {tuple(y.shape)}")
    lib = get_lib()
    (x, r, u), ctrl = _cp_prox(
        lib, _stream(dev),
        lambda xa, ra, ua, xb, rb, ub, *run: lib.dinvk_tgv_prox(_p(y), xa, ra, ua, xb, rb, ub, _p(tl1), _p(l2), B, C, H, W,
                                                                int(n_it_max), float(crit), float(tau), float(rho), *run),
        [x2, r2, u2], lib.dinvk_tgv_prox_workspace_bytes(B, C, H, W), tgv_block(lib)[1], n_it_max, check_every, stats)
    return x, r, u, torch.full((), ctrl["it_done"], dtype=torch.int32, device=dev)


def tgv_epsilon(f: torch.Tensor) -> torch.Tensor:
    """TGV's Jacobian of a vector field (B,C,H,W,2) -> (B,C,H,W,4), backward differences (tgv.py:229-270)"""
    dev = _require_cuda(f)
    if f.dim() != 5 or f.shape[-1] != 2:
        raise NotImplementedError(f"epsilon is 2-D only: expected a (B, C, H, W, 2) tensor, got {tuple(f.shape)}")
    f = _f32c(f)
    out = torch.empty((*f.shape[:-1], 4), dtype=torch.float32, device=dev)
    if f.numel():
        check(get_lib().dinvk_tv_stencil(3, _p(f), _p(out), *f.shape[:-1], _stream(dev)))
    return out


def tgv_epsilon_adjoint(g: torch.Tensor) -> torch.Tensor:
    """adjoint of `tgv_epsilon`, (B,C,H,W,4) -> (B,C,H,W,2) (tgv.py:272-312)"""
    dev = _require_cuda(g)
    if g.dim() != 5 or g.shape[-1] != 4:
        raise NotImplementedError(f"epsilon_adjoint is 2-D only: expected a (B, C, H, W, 4) tensor, got {tuple(g.shape)}")
    g = _f32c(g)
    out = torch.empty((*g.shape[:-1], 2), dtype=torch.float32, device=dev)
    if g.numel():
        check(get_lib().dinvk_tv_stencil(4, _p(g), _p(out), *g.shape[:-1], _stream(dev)))
    return out
