"""The tiled product convolution of TiledSpaceVaryingBlur (deepinv/physics/blur.py:871-1192) restated on the oracle's
blur_A / blur_At, one full-image term per patch:
    A x  = sum_k Wt_k . (h_k *valid x),   A^T y = sum_k h_k (transposed valid) (Wt_k . y),
where Wt_k is the multiplier w_k placed at patch k's origin (r s1, c s2) of the compatible grid (the image's, padded at the
bottom / right) and cropped to the valid output, which starts at (h // 2, w // 2)."""
import torch

from oracle import ref_ops as R

MODES = ["bump", "linear"]  # the fixtures' `mode` codes


def num_patches(H, W, patch, stride):
    out = []
    for n, p, s in zip((H, W), patch, stride):
        pad = (p + (abs(n - p) // s + 1) * s - n) % s
        out.append((n + pad - p) // s + 1)
    return tuple(out)


def placed(w, H, W, fh, fw, patch, stride):
    """(K, H - fh + 1, W - fw + 1): Wt_k for every k"""
    (P1, P2), (s1, s2) = patch, stride
    nr, nc = num_patches(H, W, patch, stride)
    Hc, Wc = P1 + (nr - 1) * s1, P2 + (nc - 1) * s2
    full = torch.zeros(nr * nc, max(Hc, H), max(Wc, W), dtype=w.dtype)
    for r in range(nr):
        for c in range(nc):
            full[r * nc + c, r * s1: r * s1 + P1, c * s2: c * s2 + P2] = w.reshape(-1, P1, P2)[r * nc + c]
    return full[:, fh // 2: fh // 2 + H - fh + 1, fw // 2: fw // 2 + W - fw + 1]


def tiledsv_A(x, w, h, patch, stride):
    H, W = x.shape[-2:]
    fh, fw = h.shape[-2:]
    Wt = placed(w, H, W, fh, fw, patch, stride)
    out = 0.0
    for k in range(Wt.size(0)):
        out = out + Wt[k] * R.blur_A(x, h[:, :, k], "valid")
    return out


def tiledsv_At(y, w, h, patch, stride, H, W):
    fh, fw = h.shape[-2:]
    Wt = placed(w, H, W, fh, fw, patch, stride)
    out = 0.0
    for k in range(Wt.size(0)):
        out = out + R.blur_At(Wt[k] * y, h[:, :, k], "valid", H, W)
    return out


def tiledsv_A_patches(x, w, h, patch, stride, fft=False):
    """The reference's own per-patch algorithm in torch, on any device and dtype: unfold x into halo'd patches, one valid
    convolution per patch (grouped F.conv2d of the flipped filter, or, with `fft`, a product of 2-D FFTs of the halo'd patch
    size), times w_k, fold (summing overlaps), crop to the valid output.  Filters (b, c, K, h, w) broadcast over (B, C)."""
    import torch.nn.functional as F

    B, C, H, W = x.shape
    fh, fw = h.shape[-2:]
    (P1, P2), (s1, s2) = patch, stride
    nr, nc = num_patches(H, W, patch, stride)
    K, Hc, Wc = nr * nc, P1 + (nr - 1) * s1, P2 + (nc - 1) * s2
    ai, aj = fh // 2, fw // 2
    # padded row ai + I holds compatible row I; each patch takes P1 + fh - 1 rows from its origin
    xp = F.pad(x, (aj, max(Wc, W) - W + fw - 1 - aj, ai, max(Hc, H) - H + fh - 1 - ai))
    pt = xp.unfold(2, P1 + fh - 1, s1).unfold(3, P2 + fw - 1, s2)[:, :, :nr, :nc]  # (B, C, nr, nc, P1 + fh - 1, P2 + fw - 1)
    pt = pt.reshape(B * C * K, P1 + fh - 1, P2 + fw - 1)
    hk = h.expand(B, C, K, fh, fw).reshape(B * C * K, fh, fw)
    if fft:
        L = (P1 + fh - 1, P2 + fw - 1)
        out = torch.fft.irfft2(torch.fft.rfft2(pt, s=L) * torch.fft.rfft2(hk, s=L), s=L)[:, fh - 1:, fw - 1:]
    else:
        out = F.conv2d(pt[None], torch.flip(hk, (-2, -1))[:, None], groups=B * C * K)[0]
    out = out.reshape(B * C, K, P1 * P2) * w.reshape(1, K, P1 * P2)
    y = F.fold(out.transpose(1, 2), (Hc, Wc), (P1, P2), stride=(s1, s2)).reshape(B, C, Hc, Wc)
    return y[:, :, ai: ai + H - fh + 1, aj: aj + W - fw + 1]
