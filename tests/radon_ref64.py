"""The Radon-family contracts of include/dinvk.h restated in float64 torch on the CPU.

TEST INFRASTRUCTURE ONLY.  Every function follows the C ABI (angle-major sinograms (B, C, A, P), `scale` multiplies the result),
so one restatement checks every launch path of `csrc/radon.cu` and of the ramp filter in `csrc/spectral.cu`.
tests/test_radon_ref64.py pins it to oracle/ref_ops.py (the reference's Radon / IRadon / fan beam / ramp filter) evaluated in
float64 and to the `tomo_*` / `fan_*` golden vectors.

    dinvk_radon_fwd   sino[t, j] = scale * sum_i bilinear0(x_pad, px, py)
                      px = cx + c (j - cx) + s (i - cx),  py = cx - s (j - cx) + c (i - cx),  cx = (P - 1) / 2
                      x_pad: the W x W image at offset pb of a P x P zero canvas (the inscribed disc applied first if circle)
    dinvk_radon_adj   the exact transpose of the same weights (scatter), then crop and disc
    dinvk_iradon_bp   reco = scale * sum_t bilinear0(sino as a (P x A) image, col = t, row = (T + 1) / 2 (P - 1)),
                      T = lin[x] cos - lin[y] sin on the padded grid, cropped (or disc-masked when circle)
    dinvk_fanbeam     the fan grid of radon.py:16-52, bilinear0 samples summed over the ray, and its exact transpose
    dinvk_ramp_filter out[n] = sum_m g[n - m] x[m] over the N valid samples, g[0] = 1/2, g[odd d] = -2 / (pi d)^2, else 0

cos / sin come from the fp32 angles evaluated in fp64 exactly as `Tomography._trig` does.  Angles are processed in chunks of
at most ~4 M samples, so memory stays O(P^2) per chunk.  The bilinear weights are those of grid_sample(align_corners=True,
padding_mode="zeros"): the four taps around floor(p), weights (1 - f, f), zero outside the image.
"""
from __future__ import annotations

import math

import numpy as np
import torch

F64 = torch.float64
CHUNK = 1 << 22  # samples per angle chunk


def padded_width(W: int) -> int:
    """P = ceil(sqrt(2) W) in fp32, as Tomography (radon.py:60-61)"""
    return int(((2 * torch.ones(1)).sqrt() * W).ceil())


def geometry(W: int, circle: bool):
    P = W if circle else padded_width(W)
    pb = 0 if circle else P // 2 - W // 2
    return P, pb


def trig(angles_deg):
    """(cos, sin) in fp64 of the fp32 angles, degrees -> radians as Tomography._trig / radon.py:70-71"""
    a = torch.as_tensor(angles_deg).to(torch.float32).to(F64).reshape(-1)
    th = a * 4 * torch.ones(1, dtype=F64).atan() / 180
    return th.cos(), th.sin()


def disc(W: int) -> torch.Tensor:
    """the inscribed-disc mask, evaluated in fp32 like the reference (radon.py:268-279)"""
    ax = 2 * torch.arange(W, dtype=torch.float32) / (W - 1) - 1.0
    return ((ax[None, :] ** 2 + ax[:, None] ** 2) <= 1).to(F64)


def _taps(px, py, H, Wd):
    """flat indices into an (H + 2) x (Wd + 2) canvas with a one-pixel zero border, and the four bilinear weights"""
    x0, y0 = torch.floor(px), torch.floor(py)
    wx1, wy1 = px - x0, py - y0
    ok = ((x0 >= -1) & (x0 <= Wd - 1) & (y0 >= -1) & (y0 <= H - 1)).to(F64)
    x0 = torch.where(ok > 0, x0, torch.full_like(x0, -1)).long()
    y0 = torch.where(ok > 0, y0, torch.full_like(y0, -1)).long()
    base = (y0 + 1) * (Wd + 2) + (x0 + 1)
    idx = (base, base + 1, base + Wd + 2, base + Wd + 3)
    w = ((1 - wx1) * (1 - wy1) * ok, wx1 * (1 - wy1) * ok, (1 - wx1) * wy1 * ok, wx1 * wy1 * ok)
    return idx, w


def _canvas(img):
    """(BC, H, Wd) -> (BC, (H + 2) * (Wd + 2)) with a zero border"""
    return torch.nn.functional.pad(img, (1, 1, 1, 1)).reshape(img.shape[0], -1)


def _uncanvas(acc, H, Wd):
    return acc.reshape(acc.shape[0], H + 2, Wd + 2)[:, 1:H + 1, 1:Wd + 1]


def _chunks(n, per):
    step = max(1, CHUNK // max(per, 1))
    for a in range(0, n, step):
        yield a, min(n, a + step)


def _parallel_positions(c, s, P, pb):
    """image coordinates (px - pb, py - pb) of the samples (t, i, j) of a chunk of angles"""
    cx = (P - 1) / 2
    u = torch.arange(P, dtype=F64) - cx
    J, I = u[None, None, :], u[None, :, None]
    c, s = c[:, None, None], s[:, None, None]
    return cx + c * J + s * I - pb, cx - s * J + c * I - pb


def radon_fwd(x, angles_deg, circle=False, scale=1.0):
    """dinvk_radon_fwd: (B, C, W, W) -> angle-major (B, C, A, P)"""
    B, C, W, _ = x.shape
    P, pb = geometry(W, circle)
    img = x.reshape(B * C, W, W).to(F64)
    if circle:
        img = img * disc(W)
    Z = _canvas(img)
    cos, sin = trig(angles_deg)
    out = torch.zeros(B * C, len(cos), P, dtype=F64)
    for a0, a1 in _chunks(len(cos), P * P):
        px, py = _parallel_positions(cos[a0:a1], sin[a0:a1], P, pb)
        idx, w = _taps(px, py, W, W)
        acc = 0
        for k in range(4):
            acc = acc + Z[:, idx[k].reshape(-1)].reshape(B * C, *px.shape) * w[k]
        out[:, a0:a1] = acc.sum(2)  # over the steps i
    return (out * scale).reshape(B, C, len(cos), P)


def radon_adj(y_am, angles_deg, W, circle=False, scale=1.0):
    """dinvk_radon_adj: angle-major (B, C, A, P) -> (B, C, W, W), the exact transpose of radon_fwd"""
    B, C, A, P = y_am.shape
    P_, pb = geometry(W, circle)
    assert P == P_, (P, P_)
    y = y_am.reshape(B * C, A, P).to(F64)
    cos, sin = trig(angles_deg)
    acc = torch.zeros(B * C, (W + 2) * (W + 2), dtype=F64)
    for a0, a1 in _chunks(A, P * P):
        px, py = _parallel_positions(cos[a0:a1], sin[a0:a1], P, pb)
        idx, w = _taps(px, py, W, W)
        val = y[:, a0:a1, None, :]  # ray (t, j) broadcast over its steps i
        for k in range(4):
            acc.index_add_(1, idx[k].reshape(-1), (val * w[k]).reshape(B * C, -1))
    out = _uncanvas(acc, W, W)
    if circle:
        out = out * disc(W)
    return (out * scale).reshape(B, C, W, W)


def iradon_bp(y_am, angles_deg, W, circle=False, scale=1.0):
    """dinvk_iradon_bp: IRadon.forward(filtering=False) (radon.py:396-450) without its pi / (2A), times `scale`"""
    B, C, A, P = y_am.shape
    P_, pb = geometry(W, circle)
    assert P == P_, (P, P_)
    img = y_am.reshape(B * C, A, P).to(F64).transpose(1, 2)  # the (P x A) "image": rows = detector, columns = angle
    Z = _canvas(img.contiguous())
    cos, sin = trig(angles_deg)
    lin = torch.linspace(-1, 1, P, dtype=F64)
    yg, xg = lin[pb:pb + W, None], lin[None, pb:pb + W]
    reco = torch.zeros(B * C, W, W, dtype=F64)
    for a0, a1 in _chunks(A, W * W):
        t = torch.arange(a0, a1, dtype=F64)[:, None, None]
        T = xg * cos[a0:a1, None, None] - yg * sin[a0:a1, None, None]
        X = (t * 2.0 / (A - 1) - 1.0).expand_as(T)
        idx, w = _taps((X + 1) / 2 * (A - 1), (T + 1) / 2 * (P - 1), P, A)
        for k in range(4):
            reco = reco + (Z[:, idx[k].reshape(-1)].reshape(B * C, *T.shape) * w[k]).sum(1)
    if circle:
        reco = reco * (xg ** 2 + yg ** 2 <= 1).to(F64)
    return (reco * scale).reshape(B, C, W, W)


def fan_constants(W, circle, fan_parameters=None):
    """(G, pb, D, half_len, src, den) of radon.py:16-52 / 224-240 in Python floats"""
    fp = dict(fan_parameters or {})
    fp.setdefault("pixel_spacing", 0.5 / W)
    fp.setdefault("source_radius", 57.5)
    fp.setdefault("detector_radius", 57.5)
    fp.setdefault("n_detector_pixels", 258)
    fp.setdefault("detector_spacing", 0.077)
    G, pb = geometry(W, circle)
    D = int(fp["n_detector_pixels"])
    sf = 2.0 / (G * fp["pixel_spacing"])
    src, det, sp = fp["source_radius"] * sf, fp["detector_radius"] * sf, fp["detector_spacing"] * sf
    return G, pb, D, 0.5 * sp * (D - 1), src, src + det


def _fan_positions(c, s, G, D, pb, half_len, src, den):
    xi = torch.linspace(-1, 1, G, dtype=F64)[None, None, :]  # along the ray
    yj = torch.linspace(-1, 1, D, dtype=F64)[None, :, None]  # detector
    yy = yj * (half_len * (xi + src) / den)
    c, s = c[:, None, None], s[:, None, None]
    return ((c * xi + s * yy) + 1) / 2 * (G - 1) - pb, ((-s * xi + c * yy) + 1) / 2 * (G - 1) - pb


def fanbeam_fwd(x, angles_deg, circle=False, fan_parameters=None, scale=1.0):
    """dinvk_fanbeam(adjoint=0): (B, C, W, W) -> angle-major (B, C, A, D)"""
    B, C, W, _ = x.shape
    G, pb, D, hl, src, den = fan_constants(W, circle, fan_parameters)
    img = x.reshape(B * C, W, W).to(F64)
    if circle:
        img = img * disc(W)
    Z = _canvas(img)
    cos, sin = trig(angles_deg)
    out = torch.zeros(B * C, len(cos), D, dtype=F64)
    for a0, a1 in _chunks(len(cos), G * D):
        px, py = _fan_positions(cos[a0:a1], sin[a0:a1], G, D, pb, hl, src, den)
        idx, w = _taps(px, py, W, W)
        acc = 0
        for k in range(4):
            acc = acc + Z[:, idx[k].reshape(-1)].reshape(B * C, *px.shape) * w[k]
        out[:, a0:a1] = acc.sum(3)
    return (out * scale).reshape(B, C, len(cos), D)


def fanbeam_adj(y_am, angles_deg, W, circle=False, fan_parameters=None, scale=1.0):
    """dinvk_fanbeam(adjoint=1): the exact transpose of fanbeam_fwd"""
    B, C, A, D = y_am.shape
    G, pb, D_, hl, src, den = fan_constants(W, circle, fan_parameters)
    assert D == D_, (D, D_)
    y = y_am.reshape(B * C, A, D).to(F64)
    cos, sin = trig(angles_deg)
    acc = torch.zeros(B * C, (W + 2) * (W + 2), dtype=F64)
    for a0, a1 in _chunks(A, G * D):
        px, py = _fan_positions(cos[a0:a1], sin[a0:a1], G, D, pb, hl, src, den)
        idx, w = _taps(px, py, W, W)
        val = y[:, a0:a1, :, None]
        for k in range(4):
            acc.index_add_(1, idx[k].reshape(-1), (val * w[k]).reshape(B * C, -1))
    out = _uncanvas(acc, W, W)
    if circle:
        out = out * disc(W)
    return (out * scale).reshape(B, C, W, W)


def ramp_kernel(N: int) -> np.ndarray:
    """g[d] for d = -(N-1) .. N-1: 1/2 at 0, -2 / (pi d)^2 at odd d, 0 at even d"""
    d = np.arange(-(N - 1), N, dtype=np.float64)
    g = np.where(np.abs(d) % 2 == 1, -2.0 / (math.pi * np.where(d == 0, 1.0, d)) ** 2, 0.0)
    g[N - 1] = 0.5
    return g


def ramp(y) -> torch.Tensor:
    """dinvk_ramp_filter along the last axis: the closed-form spatial sum, as a linear convolution (fp64 FFT of length >= 3N,
    which is exact to ~1e-15 of the row norm)"""
    x = torch.as_tensor(y).to(F64)
    N = x.shape[-1]
    g = ramp_kernel(N)
    L = 1
    while L < 3 * N:
        L *= 2
    X = np.fft.rfft(x.reshape(-1, N).numpy(), L, axis=-1)
    Gf = np.fft.rfft(g, L)
    full = np.fft.irfft(X * Gf, L, axis=-1)[:, N - 1:2 * N - 1]
    return torch.from_numpy(full).reshape(x.shape)


def pixel_weight_sums(theta_rad: float, u: float, v: float) -> float:
    """sum over the samples of one angle of the bilinear weights that reach one pixel: the pixel at the origin, the sample lattice
    the unit grid rotated by theta and shifted by (u, v)"""
    m = np.arange(-3, 4, dtype=np.float64)
    M, N = np.meshgrid(m, m, indexing="ij")
    c, s = math.cos(theta_rad), math.sin(theta_rad)
    px = c * M + s * N + u
    py = -s * M + c * N + v
    return float((np.maximum(0.0, 1 - np.abs(px)) * np.maximum(0.0, 1 - np.abs(py))).sum())
