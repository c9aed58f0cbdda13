"""Generate the space-varying blur golden vectors (tests/golden/svblur_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_svblur.py

Every fixture stores its inputs next to the outputs of deepinv v0.4.1's `SpaceVaryingBlur` (product_convolution2d and its
adjoint), all on CPU in float32.  `pad` is the padding's DINVK_PAD_* code (valid 0, circular 1, replicate 2, reflect 3,
constant 4).  Operator fixtures hold x, w (multipliers), h (filters), y = A x, v (a random point of A's range) and
At = A^T v; `svblur_algo` holds a CG `prox_l2` and a PGD run.
"""
from __future__ import annotations

import warnings
from pathlib import Path

import numpy as np
import torch

warnings.filterwarnings("ignore")
import deepinv as dinv  # noqa: E402  (the real reference)
from deepinv.optim import PGD  # noqa: E402
from deepinv.optim.data_fidelity import L2  # noqa: E402
from deepinv.optim.prior import Tikhonov  # noqa: E402
from deepinv.physics import SpaceVaryingBlur  # noqa: E402
from deepinv.physics.generator import MotionBlurGenerator, ProductConvolutionBlurGenerator  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
PADS = ["valid", "circular", "replicate", "reflect", "constant"]


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def operator_case(name, pad, x, w, h, use_fft=False, seed=0):
    phys = SpaceVaryingBlur(filters=h, multipliers=w, padding=pad, use_fft=use_fft)
    with torch.no_grad():
        y = phys.A(x)
        v = torch.randn(y.shape, generator=g(seed + 1))
        at = phys.A_adjoint(v)
    assert at.shape == x.shape, (name, at.shape, x.shape)
    save(name, x=x, w=w, h=h, y=y, v=v, At=at, pad=np.int32(PADS.index(pad)), use_fft=np.int32(use_fft))


def random_case(name, pad, B, C, H, W, K, fh, fw, mb, mc, fb, fc, seed):
    x = torch.randn(B, C, H, W, generator=g(seed))
    w = torch.rand(mb, mc, K, H, W, generator=g(seed + 2))
    h = torch.rand(fb, fc, K, fh, fw, generator=g(seed + 3))
    h = h / h.sum(dim=(-2, -1), keepdim=True)
    operator_case(name, pad, x, w, h, seed=seed)


def operator_fixtures():
    seed = 100
    # every padding, an odd square and an even non-square filter, K = 3 and 1, images crossing the 64-pixel tile in one
    # dimension and not a multiple of 64 in either
    for pad in PADS:
        random_case(f"svblur_{pad}_5x5_k3", pad, 2, 2, 23, 70, 3, 5, 5, 2, 2, 1, 1, seed)
        random_case(f"svblur_{pad}_4x6_k1", pad, 1, 1, 67, 21, 1, 4, 6, 1, 1, 1, 1, seed + 10)
        seed += 20
    # K = 10 with a non-square odd x even filter, both border families
    for pad in ("reflect", "circular"):
        random_case(f"svblur_{pad}_7x4_k10", pad, 1, 2, 19, 26, 10, 7, 4, 1, 2, 1, 1, seed)
        seed += 20
    # multipliers and filters broadcast over (B, C) independently: (1,1), (B,1), (1,C), (B,C) for each
    combos = {"11": (1, 1), "B1": (2, 1), "1C": (1, 3), "BC": (2, 3)}
    for i, (mn, (mb, mc)) in enumerate(combos.items()):
        for j, (fn, (fb, fc)) in enumerate(combos.items()):
            pad = PADS[(i + j) % len(PADS)]
            random_case(f"svblur_bcast_m{mn}_f{fn}", pad, 2, 3, 13, 11, 2, 3, 3, mb, mc, fb, fc, seed)
            seed += 10
    # the reference's own parameter generator: eigen-PSFs of motion blurs plus interpolated multipliers
    torch.manual_seed(7)
    pc = ProductConvolutionBlurGenerator(psf_generator=MotionBlurGenerator((9, 9), num_channels=1), img_size=(72, 66),
                                         n_eigen_psf=4, spacing=(24, 22))
    params = pc.step(1, seed=7)
    x = torch.rand(1, 1, 72, 66, generator=g(8))
    for pad in ("valid", "reflect"):
        operator_case(f"svblur_generator_{pad}", pad, x, params["multipliers"].float(), params["filters"].float(), seed=9)
    # the FFT convolutions of the reference (circular padding): the same operator up to rounding
    x = torch.randn(2, 1, 32, 40, generator=g(11))
    w = torch.rand(1, 1, 3, 32, 40, generator=g(12))
    h = torch.rand(1, 1, 3, 7, 7, generator=g(13))
    operator_case("svblur_fft_circular", "circular", x, w, h / h.sum(dim=(-2, -1), keepdim=True), use_fft=True, seed=14)


def algo_fixtures():
    x = torch.rand(1, 1, 20, 24, generator=g(20))
    w = torch.rand(1, 1, 3, 20, 24, generator=g(21))
    w = w / w.sum(dim=2, keepdim=True)
    h = torch.rand(1, 1, 3, 5, 5, generator=g(22))
    h = h / h.sum(dim=(-2, -1), keepdim=True)
    phys = SpaceVaryingBlur(filters=h, multipliers=w, padding="reflect")
    with torch.no_grad():
        y = phys.A(x) + 0.01 * torch.randn(x.shape, generator=g(23))
        z = torch.rand(x.shape, generator=g(24))
        prox = phys.prox_l2(z, y, 0.5)
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
    save("svblur_algo", x=x, w=w, h=h, y=y, z=z, gamma=np.float32(0.5), prox=prox, pgd=pgd, pad=np.int32(PADS.index("reflect")),
         max_iter=np.int32(phys.max_iter), tol=np.float64(phys.tol))


if __name__ == "__main__":
    torch.set_num_threads(1)
    operator_fixtures()
    algo_fixtures()
