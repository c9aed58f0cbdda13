"""The `dinvk_spectral` contract (include/dinvk.h, "Spectral operators") restated in complex128 torch on the CPU.

TEST INFRASTRUCTURE ONLY.  This follows the C ABI, not the reference's classes: every argument of `dinvk_spectral_args` means
here what the header says it means, so one function checks every launch path of the library (pipelined, fast tile, generic
tile, O(N^2), elementwise-only, coil reduction) against the same exact arithmetic.  tests/test_spectral_ref64.py pins it to
oracle/ref_ops.py (the reference's MRI / MultiCoilMRI / BlurFFT restated) evaluated in float64.

    u   = a0*p0 + a1*p1                          planar complex (B,2,H,W); p1 optional
    U   = F(u)               if fwd              orthonormal 2-D DFT; centred: fftshift(fft(ifftshift(.)))
    U  <- g(mask) (.) U                          DINVK_G_*; real modes scale the two planes independently
    v   = F^-1(U)            if inv
    out = e0*v + e1*q0 + e2*q1                   q0 / q1 optional
    multi-coil (ncoil > 1): coil_mode 1  u[b,n] = S[b,n] u[b], out (batch,2,ncoil,H,W)
                            coil_mode 2  out[b] = e0 * sum_n conj(S[b,n]) v[b,n]      (batch,2,H,W)
                            coil_mode 3  out[b] = sqrt(sum_n |v[b,n]|^2)              (batch,1,H,W)

The multiplier is read from the flat memory of `mask` exactly as the kernels read it: element
`mask[b*sb + ch*sc + h*sh + w]` for the real modes, the interleaved pair `((float2*)mask)[b*sb + h*sh + w]` for CMUL /
CMUL_CONJ (sc ignored), with b the batch sample (a coil image's sample for ncoil > 1); `c_batch[b]` overrides `c`.
`dtype=torch.float32` evaluates the same contract in complex64 (torch's own fp32 FFT): the yardstick of how close an fp32
evaluation can be expected to come.
"""
from __future__ import annotations

import torch

G_NONE, G_MASK, G_SQ, G_INV_SQ_PLUS_C, G_PINV, G_CMUL, G_CMUL_CONJ = range(7)
PINV_THRESHOLD = 1e-5  # DINVK_G_PINV: m > 1e-5 ? 1/m : 0


def _fft2(x: torch.Tensor, inverse: bool, centered: bool) -> torch.Tensor:
    d = (-2, -1)
    f = torch.fft.ifftn if inverse else torch.fft.fftn
    if not centered:
        return f(x, dim=d, norm="ortho")
    return torch.fft.fftshift(f(torch.fft.ifftshift(x, dim=d), dim=d, norm="ortho"), dim=d)


def _idx(nb: int, H: int, W: int, sb: int, sh: int) -> torch.Tensor:
    b = torch.arange(nb, dtype=torch.int64).view(nb, 1, 1)
    h = torch.arange(H, dtype=torch.int64).view(1, H, 1)
    w = torch.arange(W, dtype=torch.int64).view(1, 1, W)
    return b * sb + h * sh + w


def multiplier(mask: torch.Tensor, gmode: int, nb: int, H: int, W: int, strides, c: float = 0.0, c_batch=None,
               dtype=torch.float64):
    """g(mask) per batch sample: (nb,H,W) complex for CMUL / CMUL_CONJ, else a pair (g_re, g_im) of (nb,H,W) real fields"""
    sb, sc, sh = (int(s) for s in strides)
    flat = mask.detach().cpu().reshape(-1)
    i = _idx(nb, H, W, sb, sh)
    if gmode in (G_CMUL, G_CMUL_CONJ):
        m = torch.complex(flat[2 * i].to(dtype), flat[2 * i + 1].to(dtype))
        return m if gmode == G_CMUL else m.conj()
    out = []
    for ch in (0, 1):
        m = flat[i + ch * sc].to(dtype)
        if gmode == G_SQ:
            m = m * m
        elif gmode == G_INV_SQ_PLUS_C:
            cc = c_batch.detach().cpu().to(dtype).view(nb, 1, 1) if c_batch is not None else torch.tensor(c, dtype=dtype)
            m = 1.0 / (m * m + cc)
        elif gmode == G_PINV:
            m = torch.where(m > PINV_THRESHOLD, 1.0 / m, torch.zeros_like(m))
        out.append(m)
    return tuple(out)


def _cplx(planar: torch.Tensor, dtype) -> torch.Tensor:
    """(batch, 2, ...) planar -> (batch, ...) complex"""
    t = planar.detach().cpu().to(dtype)
    return torch.complex(t[:, 0], t[:, 1])


def spectral_ref(p0, H, W, *, fwd, inv, centered=True, gmode=G_NONE, mask=None, strides=(0, 0, 0), a0=1.0, p1=None, a1=0.0,
                 c=0.0, c_batch=None, q0=None, e1=0.0, q1=None, e2=0.0, e0=1.0, ncoil=0, coil_mode=0, coil_maps=None,
                 dtype=torch.float64) -> torch.Tensor:
    """the output `dinvk_spectral` must produce for these arguments (CPU tensor of `dtype`, the output's shape)"""
    nc = ncoil if ncoil > 1 else 1
    if nc > 1 and coil_mode not in (1, 2, 3):
        raise ValueError("ncoil > 1 needs coil_mode 1, 2 or 3")
    cdt = torch.complex128 if dtype == torch.float64 else torch.complex64
    # prologue: u = a0*p0 + a1*p1, as (batch, nc, H, W) complex
    if nc > 1 and coil_mode >= 2:
        batch = p0.shape[0]
        src_shape = (batch, 2, nc, H, W)
    else:
        batch = p0.numel() // (2 * H * W)
        src_shape = (batch, 2, H, W)
    u = a0 * _cplx(p0.reshape(src_shape), dtype)
    if p1 is not None:
        u = u + a1 * _cplx(p1.reshape(src_shape), dtype)
    if u.dim() == 3:
        u = u.unsqueeze(1)
    S = None
    if nc > 1 and coil_mode != 3:
        S = coil_maps.detach().cpu().to(cdt)
    if nc > 1 and coil_mode == 1:
        u = S * u                                  # (batch|1, nc) maps times the broadcast image
    U = _fft2(u, False, centered) if fwd else u
    if gmode != G_NONE:
        g = multiplier(mask, gmode, batch, H, W, strides, c, c_batch, dtype)
        if isinstance(g, tuple):
            U = torch.complex(U.real * g[0].unsqueeze(1), U.imag * g[1].unsqueeze(1))
        else:
            U = U * g.unsqueeze(1)
    v = _fft2(U, True, centered) if inv else U
    if nc > 1 and coil_mode == 2:
        r = e0 * (S.conj() * v).sum(1)
        return torch.stack([r.real, r.imag], 1)
    if nc > 1 and coil_mode == 3:
        return (v.real ** 2 + v.imag ** 2).sum(1, keepdim=True).sqrt()
    out = torch.stack([v.real, v.imag], 1)         # (batch, 2, nc, H, W)
    out = out.reshape((batch, 2, nc, H, W) if nc > 1 else tuple(p0.shape))
    out = e0 * out
    if q0 is not None:
        out = out + e1 * q0.detach().cpu().to(dtype).reshape(out.shape)
    if q1 is not None:
        out = out + e2 * q1.detach().cpu().to(dtype).reshape(out.shape)
    return out
