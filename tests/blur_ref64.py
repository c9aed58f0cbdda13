"""fp64 restatement of the direct blur contracts (csrc/blur.cu), for the launch-path table (tests/blur_path_cases.py).

  * forward (`dinvk_blur_fwd`): the image is padded explicitly by the padding's index rule (the kernel origin is (h//2, w//2); valid
    needs no padding), then the taps are summed as a true convolution over the padded image;
  * transpose (`dinvk_blur_adj`): the exact scatter of the same weights onto the extended (Ho+h-1) x (Wo+w-1) domain (a correlation of
    the explicitly zero-padded y with the unflipped filter), folded back onto the H x W image by the padding's index map (an index
    add: each extended position goes to the pixel the forward read it from; constant drops the positions outside the image).

Filters broadcast as (FB, FC) in {1, B} x {1, C}.  No step multiplies by a 0/1 mask: out-of-range taps read explicit zeros or are
left out, so a NaN or +-Inf reaches exactly the outputs whose footprint contains it, the sign of an Inf survives and +Inf + -Inf
gives NaN, as in the reference's F.pad + conv2d / conv_transpose2d.  `slow=True` sums the taps one slice at a time; the default
runs the same sums through float64 conv2d in row strips (tests/test_blur_ref64.py pins the two together).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

PADS = ("valid", "circular", "replicate", "reflect", "constant")
STRIP_ELEMS = 1 << 25  # float64 elements of one strip's im2col buffer


def map_index(e: int, n: int, pad: str):
    """the image index that extended index e reads under `pad` (None: an explicit zero); reflect and circular as the reference's
    F.pad allows them (one reflection, one wrap: e within one image size of the border)"""
    if pad == "circular":
        return e % n
    if pad == "replicate":
        return min(max(e, 0), n - 1)
    if pad == "reflect":
        r = -e if e < 0 else e
        r = 2 * (n - 1) - r if r > n - 1 else r
        assert 0 <= r < n, (e, n)
        return r
    return e if 0 <= e < n else None


def _origin(h: int) -> int:
    """rows of padding before the image: the extended domain starts at index h//2 - (h-1)"""
    return h - 1 - h // 2


def _expand(k: torch.Tensor, B: int, C: int) -> torch.Tensor:
    FB, FC = k.shape[:2]
    assert FB in (1, B) and FC in (1, C), (tuple(k.shape), B, C)
    return k.expand(B, C, *k.shape[2:])


def pad_image(x: torch.Tensor, h: int, w: int, pad: str) -> torch.Tensor:
    """(B, C, H, W) -> (B, C, H+h-1, W+w-1): the extended image the forward reads (explicit zeros for constant)"""
    H, W = x.shape[-2:]
    rows = [map_index(e - _origin(h), H, pad) for e in range(H + h - 1)]
    cols = [map_index(e - _origin(w), W, pad) for e in range(W + w - 1)]
    out = torch.zeros(*x.shape[:-2], H + h - 1, W + w - 1, dtype=x.dtype)
    ri = [i for i, r in enumerate(rows) if r is not None]
    ci = [j for j, c in enumerate(cols) if c is not None]
    src = x[..., [rows[i] for i in ri], :][..., [cols[j] for j in ci]]
    out[..., ri[0]:ri[-1] + 1, ci[0]:ci[-1] + 1] = src  # (the in-range positions are contiguous)
    return out


def valid_corr(xp: torch.Tensor, kk: torch.Tensor, slow: bool = False) -> torch.Tensor:
    """out[b, c, i, j] = sum_{u, v} kk[b, c, u, v] * xp[b, c, i + u, j + v] over the (B, C) planes (kk already expanded)"""
    B, C, Hp, Wp = xp.shape
    h, w = kk.shape[-2:]
    Ho, Wo = Hp - h + 1, Wp - w + 1
    if slow:
        out = torch.zeros(B, C, Ho, Wo, dtype=torch.float64)
        for u in range(h):
            for v in range(w):
                out = out + kk[:, :, u, v][:, :, None, None] * xp[:, :, u:u + Ho, v:v + Wo]
        return out
    n = B * C
    weight = kk.reshape(n, 1, h, w).to(torch.float64)
    src = xp.reshape(1, n, Hp, Wp).to(torch.float64)
    out = torch.empty(1, n, Ho, Wo, dtype=torch.float64)
    strip = max(1, STRIP_ELEMS // max(1, n * h * w * Wo))
    for i0 in range(0, Ho, strip):
        i1 = min(Ho, i0 + strip)
        out[:, :, i0:i1] = F.conv2d(src[:, :, i0:i1 + h - 1], weight, groups=n)
    return out.reshape(B, C, Ho, Wo)


def blur_fwd(x: torch.Tensor, k: torch.Tensor, pad: str, slow: bool = False) -> torch.Tensor:
    """A x: (B, C, H, W) -> (B, C, H-h+1, W-w+1) for valid, (B, C, H, W) otherwise"""
    x = x.to(torch.float64)
    B, C = x.shape[:2]
    h, w = k.shape[-2:]
    kk = _expand(k.to(torch.float64), B, C).flip(-2, -1)  # true convolution
    xp = x if pad == "valid" else pad_image(x, h, w, pad)
    return valid_corr(xp, kk, slow)


def fold(z: torch.Tensor, h: int, w: int, pad: str, H: int, W: int) -> torch.Tensor:
    """the transpose of pad_image: extended (B, C, H+h-1, W+w-1) -> (B, C, H, W), position e added onto map(e)"""
    rows = [map_index(e - _origin(h), H, pad) for e in range(H + h - 1)]
    cols = [map_index(e - _origin(w), W, pad) for e in range(W + w - 1)]
    ri = [i for i, r in enumerate(rows) if r is not None]
    ci = [j for j, c in enumerate(cols) if c is not None]
    t = torch.zeros(*z.shape[:-2], H, z.shape[-1], dtype=z.dtype)
    t.index_add_(-2, torch.tensor([rows[i] for i in ri]), z[..., ri, :])
    out = torch.zeros(*z.shape[:-2], H, W, dtype=z.dtype)
    out.index_add_(-1, torch.tensor([cols[j] for j in ci]), t[..., ci])
    return out


def blur_adj(y: torch.Tensor, k: torch.Tensor, pad: str, H: int, W: int, slow: bool = False) -> torch.Tensor:
    """A^T y: y of A's output shape -> (B, C, H, W)"""
    y = y.to(torch.float64)
    B, C = y.shape[:2]
    h, w = k.shape[-2:]
    kk = _expand(k.to(torch.float64), B, C)
    yp = F.pad(y, (w - 1, w - 1, h - 1, h - 1))  # explicit zeros around y
    z = valid_corr(yp, kk, slow)                 # the scatter of every y value through the weights
    return z if pad == "valid" else fold(z, h, w, pad, H, W)


def apply(call: str, inp: torch.Tensor, k: torch.Tensor, pad: str, H: int, W: int, slow: bool = False) -> torch.Tensor:
    return blur_fwd(inp, k, pad, slow) if call == "A" else blur_adj(inp, k, pad, H, W, slow)


def abs_bound(call: str, inp: torch.Tensor, k: torch.Tensor, pad: str, H: int, W: int) -> torch.Tensor:
    """the same operator on |k| and |input|: the scale of each output's rounding error"""
    return apply(call, inp.to(torch.float64).abs(), k.to(torch.float64).abs(), pad, H, W)


def _reach_fwd(s: int, n: int, h: int, pad: str) -> set:
    """forward outputs (one dimension) whose taps read image index s"""
    if pad == "valid":
        return {i for i in range(n - h + 1) if i <= s <= i + h - 1}
    return {i for i in range(n) if any(map_index(i - u + h // 2, n, pad) == s for u in range(h))}


def footprint(call: str, pad: str, H: int, W: int, h: int, w: int, p: int, q: int) -> torch.Tensor:
    """boolean mask of the outputs that input pixel (p, q) reaches, from index arithmetic alone: for A, the outputs (A's shape)
    whose taps read x[p, q]; for A^T, the image pixels s (H x W) whose forward outputs include y[p, q]"""
    if call == "A":
        rows, cols = _reach_fwd(p, H, h, pad), _reach_fwd(q, W, w, pad)
        Ho, Wo = (H - h + 1, W - w + 1) if pad == "valid" else (H, W)
    else:
        rows = {s for s in range(H) if p in _reach_fwd(s, H, h, pad)}
        cols = {s for s in range(W) if q in _reach_fwd(s, W, w, pad)}
        Ho, Wo = H, W
    m = torch.zeros(Ho, Wo, dtype=torch.bool)
    if rows and cols:
        m[torch.tensor(sorted(rows))[:, None], torch.tensor(sorted(cols))[None, :]] = True
    return m
