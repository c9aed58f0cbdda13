"""Filter constructors used by Blur / BlurFFT / Downsampling (deepinv/physics/functional/blur.py:137-372,552-583), the
product convolution of SpaceVaryingBlur (deepinv/physics/functional/product_convolution.py:10-68), and the patch geometry and
blending multipliers of TiledSpaceVaryingBlur (deepinv/utils/_tiling.py:12-61, functional/tiled_product_convolution.py).

Filter generation is host-side (a few hundred taps): plain torch on whatever device is asked for; the operators that
consume these filters, and the product convolution itself, run on the libdinvk kernels."""
from __future__ import annotations

from math import exp, pi, sqrt

import torch

from .imresize import imresize_matlab  # noqa: F401


def gaussian_blur(psf_size=None, sigma=(1.0, 1.0), angle=0.0, device="cpu", dtype=torch.float32) -> torch.Tensor:
    """2-D anisotropic, rotated Gaussian kernels (B,1,h,w), each normalised to sum 1 (functional/blur.py:137-264).
    sigma: float | (sy, sx) | (B,2) tensor in (height, width) order; angle: degrees, float | (B,) tensor."""
    if isinstance(sigma, (int, float)):
        sigma = (float(sigma), float(sigma))
    sig = torch.as_tensor(sigma, device=device, dtype=dtype)
    if sig.dim() == 1:
        sig = sig[None]
    if sig.shape[-1] != 2:
        raise ValueError("deepinv_b200.gaussian_blur: 2-D kernels only (sigma = (sy, sx))")
    ang = torch.as_tensor(angle, device=device, dtype=dtype).reshape(-1)
    B = max(sig.shape[0], ang.numel())
    sig, ang = sig.expand(B, 2), ang.expand(B)
    if psf_size is None:
        c = int(float(sig.max()) / 0.3 + 1)
        psf_size = (2 * c + 1, 2 * c + 1)
    h, w = psf_size
    ay = torch.linspace(-((h - 1) / 2), (h - 1) / 2, h, device=device, dtype=dtype)
    ax = torch.linspace(-((w - 1) / 2), (w - 1) / 2, w, device=device, dtype=dtype)
    yy, xx = torch.meshgrid(ay, ax, indexing="ij")
    coords = torch.stack([xx, yy], dim=-1)[None].expand(B, h, w, 2)
    th = ang * (pi / 180.0)
    rot = torch.stack([torch.cos(th), -torch.sin(th), torch.sin(th), torch.cos(th)], dim=1).view(B, 2, 2)
    coords = torch.einsum("bij,b...j->b...i", rot, coords)
    sxy = torch.flip(sig, dims=(1,))  # (sx, sy)
    kernel = torch.ones((B, h, w), device=device, dtype=dtype)
    for d in range(2):
        s = sxy[:, d].view(B, 1, 1)
        kernel = kernel * torch.exp(-0.5 * coords[..., d] ** 2 / s ** 2) / (sqrt(2 * pi) * s)
    kernel = kernel / kernel.sum(dim=(1, 2), keepdim=True)
    return kernel[:, None]


def kaiser_window(beta: float, length: int, device="cpu") -> torch.Tensor:
    if beta < 0:
        raise ValueError("beta must be greater than 0")
    if length < 1:
        raise ValueError("length must be greater than 0")
    if length == 1:
        return torch.tensor([1.0])
    half = (length - 1) / 2
    n = torch.arange(length, device=device)
    beta = torch.tensor(beta, device=device)
    return torch.i0(beta * torch.sqrt(1 - ((n - half) / half) ** 2)) / torch.i0(beta)


def sinc_filter(factor=2, length: int = 11, windowed: bool = True, device="cpu") -> torch.Tensor:
    """separable anti-aliasing sinc, optionally Kaiser-windowed (functional/blur.py:283-336)"""
    if isinstance(factor, torch.Tensor):
        factor = factor.cpu().item()
    deltaf = 2 * (2 - 1.4142136) / factor
    n = torch.arange(length, device=device) - (length - 1) / 2
    f = torch.sinc(n / factor)
    if windowed:
        A = 2.285 * (length - 1) * 3.14159 * deltaf + 7.95
        beta = 0 if A <= 21 else (0.5842 * (A - 21) ** 0.4 + 0.07886 * (A - 21) if A <= 50 else 0.1102 * (A - 8.7))
        f = f * kaiser_window(beta, length, device=device)
    f = f.unsqueeze(0)
    f = (f * f.T)[None, None]
    return f / f.sum()


def bilinear_filter(factor: int = 2, device="cpu") -> torch.Tensor:
    """(2 factor)^2 tent filter (functional/blur.py:339-366)"""
    if isinstance(factor, torch.Tensor):
        factor = factor.cpu().item()
    x = torch.arange(start=-factor + 0.5, end=factor, step=1, device=device) / factor
    w = 1 - x.abs()
    w = torch.outer(w, w)
    return (w / w.sum())[None, None]


def bicubic_filter(factor: int = 2, device="cpu") -> torch.Tensor:
    """(4 factor)^2 Keys cubic, a = -0.5 (functional/blur.py:552-583)"""
    if isinstance(factor, torch.Tensor):
        factor = factor.cpu().item()
    x = (torch.arange(start=-2 * factor + 0.5, end=2 * factor, step=1, device=device) / factor).abs()
    a = -0.5
    w = ((a + 2) * x.pow(3) - (a + 3) * x.pow(2) + 1) * (x <= 1)
    w = w + (a * x.pow(3) - 5 * a * x.pow(2) + 8 * a * x - 4 * a) * (x > 1) * (x < 2)
    w = torch.outer(w, w)
    return (w / w.sum())[None, None]


def _product_convolution_args(t: torch.Tensor, w: torch.Tensor, h: torch.Tensor, padding: str, H: int, W: int):
    """the reference's failure modes, then the filters cut to the K terms the multipliers define"""
    from .blur import _check_filter, _padding_code

    code = _padding_code(padding)
    if t.dim() != 4:
        raise ValueError(f"Expected Tensor dimension to be 4 (2-D blur), is {t.dim()}")
    K = w.size(2)
    if h.size(2) < K:  # the reference indexes h[:, :, k] for every k < K
        raise IndexError(f"index {h.size(2)} is out of bounds for dimension 2 with size {h.size(2)}")
    h = h[:, :, :K]
    B, C = t.shape[:2]
    _check_filter(h, B, C)
    # the reference multiplies x (B, C, H, W) by w[:, :, k]: a shape that does not broadcast raises torch's RuntimeError
    if torch.broadcast_shapes((B, C, H, W), w[:, :, 0].shape) != (B, C, H, W):
        raise RuntimeError(f"multipliers of shape {tuple(w.shape)} do not broadcast to images of shape {(B, C, H, W)}")
    if tuple(w.shape[-2:]) != (H, W):
        w = w.expand(*w.shape[:3], H, W)
    return w, h, code


def product_convolution2d(x: torch.Tensor, w: torch.Tensor, h: torch.Tensor, padding: str = "valid",
                          use_fft: bool = False) -> torch.Tensor:
    r"""y = sum_k h_k * (w_k . x) (product_convolution.py:10-41): x (B, C, H, W), multipliers w (b, c, K, H, W), filters
    h (b', c', K, h, w), b, b' in {1, B} and c, c' in {1, C}.  One fused kernel (`dinvk_svblur_fwd`) for every padding;
    `use_fft` selects the reference's FFT convolutions, the same operator up to rounding, and runs the same kernel here."""
    from .. import ops
    from .forward import linear_apply

    H, W = x.shape[-2:]
    w, h, code = _product_convolution_args(x, w, h, padding, H, W)
    return linear_apply(x, lambda t: ops.svblur_fwd(t, w, h, code), lambda t: ops.svblur_adj(t, w, h, code, H, W))


def product_convolution2d_adjoint(y: torch.Tensor, w: torch.Tensor, h: torch.Tensor, padding: str = "valid",
                                  use_fft: bool = False) -> torch.Tensor:
    r"""x = sum_k w_k . (h_k^T * y) (product_convolution.py:44-68), one fused kernel (`dinvk_svblur_adj`).  The image size
    follows from y and h as in the reference: (H + h - 1, W + w - 1) for valid padding, y's own size otherwise."""
    from .. import ops
    from .forward import linear_apply

    if y.dim() != 4:
        raise ValueError(f"Expected Tensor dimension to be 4 (2-D blur), is {y.dim()}")
    fh, fw = h.shape[-2:]
    H, W = (y.shape[-2] + fh - 1, y.shape[-1] + fw - 1) if padding.lower() == "valid" else tuple(y.shape[-2:])
    w, h, code = _product_convolution_args(y, w, h, padding, H, W)
    return linear_apply(y, lambda t: ops.svblur_adj(t, w, h, code, H, W), lambda t: ops.svblur_fwd(t, w, h, code))


# ---- tiled space-varying blur: patch geometry (deepinv/utils/_tiling.py:12-61) and multipliers --------------------------------
def _as_pair(v) -> tuple[int, int]:
    return (v, v) if isinstance(v, int) else tuple(v)


def _resolve_tiling_params(patch_size, stride=None) -> tuple[tuple[int, int], tuple[int, int]]:
    patch_size = _as_pair(patch_size)
    stride = _as_pair(stride) if stride is not None else tuple(p // 2 for p in patch_size)
    if stride[0] > patch_size[0] or stride[1] > patch_size[1]:
        raise ValueError(f"Stride {stride} must be smaller or equal than patch_size {patch_size}.")
    return patch_size, stride


def _needed_pad(img_size, patch_size, stride) -> tuple[int, int]:
    """rows / columns of zeros added at the bottom / right so that the patches tile the image"""
    return tuple((p + (abs(n - p) // s + 1) * s - n) % s for n, p, s in zip(img_size, patch_size, stride))


def _compatible_size(img_size, patch_size, stride) -> tuple[int, int]:
    return tuple(n + d for n, d in zip(img_size, _needed_pad(img_size, patch_size, stride)))


def _num_patches(img_size, patch_size, stride) -> tuple[int, int]:
    return tuple((n - p) // s + 1 for n, p, s in zip(_compatible_size(img_size, patch_size, stride), patch_size, stride))


def bump_function(x: torch.Tensor, a: float = 1.0, b: float = 1.0) -> torch.Tensor:
    """1 on [-a, a], a smooth bump down to 0 on [-a-b, -a] and [a, a+b] (deepinv/physics/generator/blur.py:1014-1047)"""
    abs_x = torch.abs(x)
    t = (abs_x - a) / b
    safe_t = t.clamp(0.0, 1.0 - 1e-6)
    transition = torch.exp(-1.0 / (1.0 - safe_t ** 2)) / exp(-1.0)
    return torch.where(abs_x <= a, 1.0, torch.where(abs_x < a + b, transition, 0.0))


def _unity_partition_1d(n: int, patch: int, stride: int, mode: str, dtype) -> torch.Tensor:
    """(n_patch, n) masks summing to 1 along each column (tiled_product_convolution.py:9-59)"""
    n_patch = (n - patch) // stride + 1
    max_size = patch + (n_patch - 1) * stride
    overlap = patch - stride
    t = torch.linspace(-max_size // 2, max_size // 2, max_size, dtype=dtype)
    if mode.lower() == "bump":
        mask = bump_function(t, patch / 2 - overlap, overlap).roll(shifts=-max_size // 2 + patch // 2)
    elif mode.lower() == "linear":
        a, b = patch / 2 - overlap, overlap
        mask = ((a + b) / b - t.abs().clip(0, a + b) / b).abs().clip(0, 1)  # b = 0 (stride == patch): ZeroDivisionError
        mask = mask.roll(shifts=-max_size // 2 + patch // 2)
    else:
        raise ValueError(f"Unknown mode: {mode}. Use 'bump' or 'linear'.")
    masks = torch.stack([mask.roll(shifts=stride * i) for i in range(n_patch)], dim=0)
    masks[0, :stride] = 1.0
    masks[-1, -stride:] = 1.0
    return masks / (masks.sum(dim=0, keepdims=True) + 1e-8)


def generate_tiled_multipliers(img_size, patch_size, stride, mode: str = "bump", device="cpu",
                               dtype=torch.float32) -> torch.Tensor:
    r"""The blending multipliers of TiledSpaceVaryingBlur, (1, 1, K, P1, P2) (tiled_product_convolution.py:105-143): the outer
    product of two 1-D partitions of unity, renormalised over the K patches, cut to each patch.  Host-side parameter
    generation: evaluated on the CPU in `dtype` with the reference's operations (so float32 gives the reference's CPU values bit
    for bit), then copied to `device` once.  The normaliser is the reference's sum over the (nr, nc, H, W) product, which takes
    4 K H W bytes of host memory for a moment."""
    img_size, patch_size, stride = _as_pair(img_size), _as_pair(patch_size), _as_pair(stride)
    mx = _unity_partition_1d(img_size[0], patch_size[0], stride[0], mode, dtype)
    my = _unity_partition_1d(img_size[1], patch_size[1], stride[1], mode, dtype)
    masks = torch.tensordot(mx, my, dims=0).permute(0, 2, 1, 3)
    norm = masks.sum(dim=(0, 1)) + 1e-8
    (P1, P2), (s1, s2) = patch_size, stride
    w = torch.stack([masks[i, j, i * s1: i * s1 + P1, j * s2: j * s2 + P2] / norm[i * s1: i * s1 + P1, j * s2: j * s2 + P2]
                     for i in range(mx.size(0)) for j in range(my.size(0))])
    return w[None, None].to(device)
