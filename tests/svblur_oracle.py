"""The product convolution of SpaceVaryingBlur (deepinv/physics/functional/product_convolution.py:10-68) restated on the
oracle's blur_A / blur_At: one full multiply + blur per term, summed in k order, as the reference loops."""
import torch

from oracle import ref_ops as R

PADS = ["valid", "circular", "replicate", "reflect", "constant"]  # DINVK_PAD_* order (the fixtures' `pad` codes)


def svblur_A(x: torch.Tensor, w: torch.Tensor, h: torch.Tensor, padding: str = "valid") -> torch.Tensor:
    out = 0.0
    for k in range(w.size(2)):
        out = out + R.blur_A(w[:, :, k] * x, h[:, :, k], padding)
    return out


def svblur_At(y: torch.Tensor, w: torch.Tensor, h: torch.Tensor, padding: str, H: int, W: int) -> torch.Tensor:
    out = 0.0
    for k in range(w.size(2)):
        out = out + w[:, :, k] * R.blur_At(y, h[:, :, k], padding, H, W)
    return out
