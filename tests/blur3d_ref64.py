"""fp64 restatement of the 3-D blur contracts (csrc/blur.cu: `dinvk_blur3d_fwd` / `dinvk_blur3d_adj`), for the launch-path table
(tests/blur3d_path_cases.py) and the golden checks (tests/test_blur3d_ref64.py).

  * forward: the volume is padded explicitly along each axis by the padding's index rule (kernel origin (d//2, h//2, w//2); valid
    needs no padding), then the taps are summed as a true convolution over the padded volume;
  * transpose: the exact scatter of the same weights onto the extended (Do+d-1, Ho+h-1, Wo+w-1) domain (a correlation of the
    explicitly zero-padded y with the unflipped filter), folded back onto the D x H x W volume by the per-axis index maps, one axis
    after the other (each extended position goes to the voxel the forward read it from; constant drops positions outside).

The index rule per axis is tests/blur_ref64.py's `map_index`.  No step multiplies by a 0/1 mask, so a NaN or +-Inf reaches exactly
the outputs whose footprint contains it.  `slow=True` sums the taps one shifted slice at a time; the default runs the same sums
through float64 conv3d in depth slabs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from blur_ref64 import PADS, _expand, _origin, map_index  # noqa: F401  (PADS re-exported)

SLAB_ELEMS = 1 << 25  # float64 elements of one slab's im2col buffer


def _maps(n: int, f: int, pad: str):
    """(extended positions that read the volume, the index each reads) along one axis of length n, filter extent f"""
    m = [map_index(e - _origin(f), n, pad) for e in range(n + f - 1)]
    keep = [e for e, r in enumerate(m) if r is not None]
    return keep, [m[e] for e in keep]


def pad_volume(x: torch.Tensor, d: int, h: int, w: int, pad: str) -> torch.Tensor:
    """(B, C, D, H, W) -> (B, C, D+d-1, H+h-1, W+w-1): the extended volume the forward reads (explicit zeros for constant)"""
    out = x
    for axis, f in ((-3, d), (-2, h), (-1, w)):
        n = out.shape[axis]
        keep, src = _maps(n, f, pad)
        shape = list(out.shape)
        shape[axis] = n + f - 1
        ext = torch.zeros(shape, dtype=out.dtype)
        ext.index_copy_(axis % ext.dim(), torch.tensor(keep), out.index_select(axis % out.dim(), torch.tensor(src)))
        out = ext
    return out


def valid_corr(xp: torch.Tensor, kk: torch.Tensor, slow: bool = False) -> torch.Tensor:
    """out[b, c, z, i, j] = sum_{t, u, v} kk[b, c, t, u, v] * xp[b, c, z + t, i + u, j + v] (kk already expanded)"""
    B, C, Dp, Hp, Wp = xp.shape
    d, h, w = kk.shape[-3:]
    Do, Ho, Wo = Dp - d + 1, Hp - h + 1, Wp - w + 1
    if slow:
        out = torch.zeros(B, C, Do, Ho, Wo, dtype=torch.float64)
        for t in range(d):
            for u in range(h):
                for v in range(w):
                    out = out + kk[:, :, t, u, v][:, :, None, None, None] * xp[:, :, t:t + Do, u:u + Ho, v:v + Wo]
        return out
    n = B * C
    weight = kk.reshape(n, 1, d, h, w).to(torch.float64)
    src = xp.reshape(1, n, Dp, Hp, Wp).to(torch.float64)
    out = torch.empty(1, n, Do, Ho, Wo, dtype=torch.float64)
    slab = max(1, SLAB_ELEMS // max(1, n * d * h * w * Ho * Wo))
    for z0 in range(0, Do, slab):
        z1 = min(Do, z0 + slab)
        out[:, :, z0:z1] = F.conv3d(src[:, :, z0:z1 + d - 1], weight, groups=n)
    return out.reshape(B, C, Do, Ho, Wo)


def blur3d_fwd(x: torch.Tensor, k: torch.Tensor, pad: str, slow: bool = False) -> torch.Tensor:
    """A x: (B, C, D, H, W) -> (B, C, D-d+1, H-h+1, W-w+1) for valid, (B, C, D, H, W) otherwise"""
    x = x.to(torch.float64)
    B, C = x.shape[:2]
    d, h, w = k.shape[-3:]
    kk = _expand(k.to(torch.float64), B, C).flip(-3, -2, -1)  # true convolution
    xp = x if pad == "valid" else pad_volume(x, d, h, w, pad)
    return valid_corr(xp, kk, slow)


def fold(z: torch.Tensor, d: int, h: int, w: int, pad: str, D: int, H: int, W: int) -> torch.Tensor:
    """the transpose of pad_volume: extended (B, C, D+d-1, H+h-1, W+w-1) -> (B, C, D, H, W), one axis at a time"""
    out = z
    for axis, f, n in ((-1, w, W), (-2, h, H), (-3, d, D)):
        keep, dst = _maps(n, f, pad)
        shape = list(out.shape)
        shape[axis] = n
        t = torch.zeros(shape, dtype=out.dtype)
        t.index_add_(axis % t.dim(), torch.tensor(dst), out.index_select(axis % out.dim(), torch.tensor(keep)))
        out = t
    return out


def blur3d_adj(y: torch.Tensor, k: torch.Tensor, pad: str, D: int, H: int, W: int, slow: bool = False) -> torch.Tensor:
    """A^T y: y of A's output shape -> (B, C, D, H, W)"""
    y = y.to(torch.float64)
    B, C = y.shape[:2]
    d, h, w = k.shape[-3:]
    kk = _expand(k.to(torch.float64), B, C)
    yp = F.pad(y, (w - 1, w - 1, h - 1, h - 1, d - 1, d - 1))  # explicit zeros around y
    z = valid_corr(yp, kk, slow)                                 # the scatter of every y value through the weights
    return z if pad == "valid" else fold(z, d, h, w, pad, D, H, W)


def apply(call: str, inp: torch.Tensor, k: torch.Tensor, pad: str, D: int, H: int, W: int, slow: bool = False) -> torch.Tensor:
    return blur3d_fwd(inp, k, pad, slow) if call == "A" else blur3d_adj(inp, k, pad, D, H, W, slow)


def abs_bound(call: str, inp: torch.Tensor, k: torch.Tensor, pad: str, D: int, H: int, W: int) -> torch.Tensor:
    """the same operator on |k| and |input|: the scale of each output's rounding error"""
    return apply(call, inp.to(torch.float64).abs(), k.to(torch.float64).abs(), pad, D, H, W)
