"""The `dinvk_spectral3d` contract (include/dinvk.h) restated in complex128 torch on the CPU.

TEST INFRASTRUCTURE ONLY.  Like tests/spectral_ref64.py, this follows the C ABI rather than the reference's classes, with the 3-D
transform (fftn over (D,H,W) with the centring shifts) and the depth-aware addressing of the multiplier:

    u   = a0*p0 + a1*p1                          planar complex (B,2,D,H,W); p1 optional
    U   = F3(u)              if fwd              orthonormal 3-D DFT; centred: fftshift(fftn(ifftshift(.)))
    U  <- g(mask) (.) U                          g read at mask[b*sb + ch*sc + (d*H + h)*sh + w]
    v   = F3^-1(U)           if inv
    out = e0*v + e1*q0 + e2*q1
    no coils (coil_mode 0), ncoil = N > 1:  p0 / p1 / q0 / q1 / out (batch,2,N,D,H,W), volume by volume, mask of sample b
    coils (coil_mode 1..3, any ncoil >= 1): 1  u[b,n] = S[b,n] u[b], out (batch,2,ncoil,D,H,W)
                                            2  out[b] = e0 * sum_n conj(S[b,n]) v[b,n]      (batch,2,D,H,W)
                                            3  out[b] = sqrt(sum_n |v[b,n]|^2)              (batch,1,D,H,W)

tests/test_mri3d_ref64.py pins it to oracle/ref_ops.py's 3-D transform in float64 and to the mri3d_* golden vectors of the real
reference.  `dtype=torch.float32` evaluates the same contract in complex64 (torch's own fp32 FFT).
"""
from __future__ import annotations

import torch

G_NONE, G_MASK, G_SQ, G_INV_SQ_PLUS_C, G_PINV, G_CMUL, G_CMUL_CONJ = range(7)
PINV_THRESHOLD = 1e-5


def fft3(x: torch.Tensor, inverse: bool, centered: bool = True) -> torch.Tensor:
    d = (-3, -2, -1)
    f = torch.fft.ifftn if inverse else torch.fft.fftn
    if not centered:
        return f(x, dim=d, norm="ortho")
    return torch.fft.fftshift(f(torch.fft.ifftshift(x, dim=d), dim=d, norm="ortho"), dim=d)


def multiplier(mask, gmode, nb, D, H, W, strides, c=0.0, c_batch=None, dtype=torch.float64):
    """g(mask) per batch sample: (nb,D,H,W) complex for CMUL / CMUL_CONJ, else a pair (g_re, g_im) of (nb,D,H,W) real fields"""
    sb, sc, sh = (int(s) for s in strides)
    flat = mask.detach().cpu().reshape(-1)
    b = torch.arange(nb, dtype=torch.int64).view(nb, 1, 1, 1)
    d = torch.arange(D, dtype=torch.int64).view(1, D, 1, 1)
    h = torch.arange(H, dtype=torch.int64).view(1, 1, H, 1)
    w = torch.arange(W, dtype=torch.int64).view(1, 1, 1, W)
    i = b * sb + (d * H + h) * sh + w
    if gmode in (G_CMUL, G_CMUL_CONJ):
        m = torch.complex(flat[2 * i].to(dtype), flat[2 * i + 1].to(dtype))
        return m if gmode == G_CMUL else m.conj()
    out = []
    for ch in (0, 1):
        m = flat[i + ch * sc].to(dtype)
        if gmode == G_SQ:
            m = m * m
        elif gmode == G_INV_SQ_PLUS_C:
            cc = c_batch.detach().cpu().to(dtype).view(nb, 1, 1, 1) if c_batch is not None else torch.tensor(c, dtype=dtype)
            m = 1.0 / (m * m + cc)
        elif gmode == G_PINV:
            m = torch.where(m > PINV_THRESHOLD, 1.0 / m, torch.zeros_like(m))
        out.append(m)
    return tuple(out)


def _cplx(planar: torch.Tensor, dtype) -> torch.Tensor:
    t = planar.detach().cpu().to(dtype)
    return torch.complex(t[:, 0], t[:, 1])


def spectral3d_ref(p0, D, H, W, *, fwd, inv, centered=True, gmode=G_NONE, mask=None, strides=(0, 0, 0), a0=1.0, p1=None, a1=0.0,
                   c=0.0, c_batch=None, q0=None, e1=0.0, q1=None, e2=0.0, e0=1.0, ncoil=0, coil_mode=0, coil_maps=None,
                   dtype=torch.float64) -> torch.Tensor:
    """the output `dinvk_spectral3d` must produce for these arguments (CPU tensor of `dtype`, the output's shape)"""
    nc = max(int(ncoil), 1)
    cdt = torch.complex128 if dtype == torch.float64 else torch.complex64
    if coil_mode >= 2 or (coil_mode == 0 and nc > 1):  # y (batch,2,ncoil,D,H,W), or a plain stack of ncoil volumes per sample
        batch = p0.shape[0]
        src_shape = (batch, 2, nc, D, H, W)
    else:
        batch = p0.numel() // (2 * D * H * W)
        src_shape = (batch, 2, D, H, W)
    u = a0 * _cplx(p0.reshape(src_shape), dtype)
    if p1 is not None:
        u = u + a1 * _cplx(p1.reshape(src_shape), dtype)
    if u.dim() == 4:
        u = u.unsqueeze(1)                         # (batch, nc, D, H, W)
    S = coil_maps.detach().cpu().to(cdt) if coil_mode in (1, 2) else None
    if coil_mode == 1:
        u = S * u
    U = fft3(u, False, centered) if fwd else u
    if gmode != G_NONE:
        g = multiplier(mask, gmode, batch, D, H, W, strides, c, c_batch, dtype)
        if isinstance(g, tuple):
            U = torch.complex(U.real * g[0].unsqueeze(1), U.imag * g[1].unsqueeze(1))
        else:
            U = U * g.unsqueeze(1)
    v = fft3(U, True, centered) if inv else U
    if coil_mode == 2:
        r = e0 * (S.conj() * v).sum(1)
        return torch.stack([r.real, r.imag], 1)
    if coil_mode == 3:
        return (v.real ** 2 + v.imag ** 2).sum(1, keepdim=True).sqrt()
    out = torch.stack([v.real, v.imag], 1)         # (batch, 2, nc, D, H, W)
    out = out.reshape((batch, 2, nc, D, H, W) if coil_mode == 1 or nc > 1 else tuple(p0.shape))
    out = e0 * out
    if q0 is not None:
        out = out + e1 * q0.detach().cpu().to(dtype).reshape(out.shape)
    if q1 is not None:
        out = out + e2 * q1.detach().cpu().to(dtype).reshape(out.shape)
    return out


# the reference's operators, written with the restatement (what the mri3d_* fixtures hold, evaluated in float64)
def full_mask(mask):
    """(B|1,2,D,H,W) mask -> (tensor, strides) in the ABI's addressing"""
    B, _, D, H, W = mask.shape
    return mask.contiguous(), (2 * D * H * W if B > 1 else 0, D * H * W, W)


def mc_A(x, mask, maps):
    mt, st = full_mask(mask)
    return spectral3d_ref(x, *x.shape[-3:], fwd=True, inv=False, gmode=G_MASK, mask=mt, strides=st, ncoil=maps.shape[1],
                          coil_mode=1, coil_maps=maps)


def mc_At(y, mask, maps, rss=False):
    mt, st = full_mask(mask)
    return spectral3d_ref(y, *y.shape[-3:], fwd=False, inv=True, gmode=G_MASK, mask=mt, strides=st, ncoil=y.shape[2],
                          coil_mode=3 if rss else 2, coil_maps=maps)
