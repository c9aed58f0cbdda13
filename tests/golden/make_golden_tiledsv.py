"""Generate the tiled space-varying blur golden vectors (tests/golden/tiledsv_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_tiledsv.py

Every fixture stores the inputs and outputs of deepinv v0.4.1's `TiledSpaceVaryingBlur`, on CPU in float32: x, h (filters),
w (the reference's multipliers, (1, 1, K, P1, P2)), y = A x, v (a random point of A's range) and At = A^T v, with the
patch, stride, blending mode (0 bump, 1 linear) and use_fft.  `tiledsv_algo` holds a CG `prox_l2` and a PGD run.
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
from deepinv.physics import TiledSpaceVaryingBlur  # noqa: E402
from deepinv.physics.functional import bilinear_filter  # noqa: E402
from deepinv.physics.generator import MotionBlurGenerator, TiledBlurGenerator  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
MODES = ["bump", "linear"]  # the fixtures' `mode` codes


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def operator_case(name, x, h, patch, stride, mode="bump", use_fft=True, seed=0):
    phys = TiledSpaceVaryingBlur(filters=h, patch_size=patch, stride=stride, blending_mode=mode, use_fft=use_fft)
    with torch.no_grad():
        y = phys.A(x)
        v = torch.randn(y.shape, generator=g(seed + 1))
        at = phys.A_adjoint(v)
    assert at.shape == x.shape, (name, at.shape, x.shape)
    save(name, x=x, h=h, w=phys.multipliers, y=y, v=v, At=at, patch=np.int32(pair(patch)), stride=np.int32(pair(stride)),
         mode=np.int32(MODES.index(mode)), use_fft=np.int32(use_fft))


def random_case(name, B, C, H, W, fh, fw, patch, stride, fb=1, fc=1, mode="bump", use_fft=True, seed=0):
    nr, nc = TiledSpaceVaryingBlur.num_filters((H, W), patch, stride)
    x = torch.randn(B, C, H, W, generator=g(seed))
    h = torch.rand(fb, fc, nr * nc, fh, fw, generator=g(seed + 3))
    operator_case(name, x, h / h.sum(dim=(-2, -1), keepdim=True), patch, stride, mode, use_fft, seed)


def operator_fixtures():
    # the reference's own test case: bilinear_filter(2) on every patch
    x = torch.randn(1, 3, 20, 13, generator=g(1))
    nr, nc = TiledSpaceVaryingBlur.num_filters((20, 13), (8, 5), (4, 3))
    h = bilinear_filter(2).unsqueeze(2).repeat(1, 1, nr * nc, 1, 1)
    operator_case("tiledsv_reference_case", x, h, (8, 5), (4, 3), seed=2)
    # a subset of the reference's adjointness grid, both blending modes and both convolution paths
    seed = 100
    grid = [((32, 32), 8, 4, (5, 5)), ((33, 33), 9, 5, (6, 6)), ((32, 33), (8, 9), (4, 5), (5, 6)), ((33, 33), 8, (4, 5), (6, 6)),
            ((32, 33), (8, 9), 5, (5, 5))]
    for i, (size, patch, stride, psf) in enumerate(grid):
        for mode in ("bump", "linear"):
            use_fft = (i + (mode == "linear")) % 2 == 0
            random_case(f"tiledsv_grid{i}_{mode}", 2, 1, *size, *psf, patch, stride, mode=mode, use_fft=use_fft, seed=seed)
            seed += 10
    # the four filter broadcasts
    for fn, (fb, fc) in {"11": (1, 1), "B1": (2, 1), "1C": (1, 3), "BC": (2, 3)}.items():
        random_case(f"tiledsv_bcast_f{fn}", 2, 3, 29, 27, 5, 4, 10, 6, fb=fb, fc=fc, seed=seed)
        seed += 10
    # patch not a multiple of the stride, compatible-size padding (230 -> 240 rows, 197 -> 240 columns: the last patch row and
    # column reach into it), 4 x 4 or more 64-pixel tiles in both directions.  The inputs are dyadic (x and v multiples of 1/64
    # and 1/32, taps multiples of 1/256 summing to 1) and the convolution direct, so the stored arrays compress well.
    nr, nc = TiledSpaceVaryingBlur.num_filters((230, 197), (100, 90), (70, 50))
    assert (nr, nc) == (3, 4)
    x = torch.randint(0, 64, (1, 1, 230, 197), generator=g(seed)) / 64.0
    counts = torch.stack([torch.multinomial(torch.ones(49), 256, replacement=True, generator=g(seed + 3 + k)).bincount(minlength=49)
                          for k in range(nr * nc)])
    h = (counts.float() / 256.0).reshape(1, 1, nr * nc, 7, 7)
    phys = TiledSpaceVaryingBlur(filters=h, patch_size=(100, 90), stride=(70, 50), use_fft=False)
    with torch.no_grad():
        y = phys.A(x)
        v = torch.randint(-32, 33, y.shape, generator=g(seed + 1)) / 32.0
        at = phys.A_adjoint(v)
    save("tiledsv_large_pad", x=x, h=h, w=phys.multipliers, y=y, v=v, At=at, patch=np.int32((100, 90)),
         stride=np.int32((70, 50)), mode=np.int32(0), use_fft=np.int32(0))
    # an image smaller than the patch; stride == patch (bump: all-ones multipliers)
    random_case("tiledsv_small_image", 1, 2, 10, 12, 3, 3, 16, 8, seed=seed + 10)
    random_case("tiledsv_stride_eq_patch", 1, 1, 40, 36, 5, 5, (20, 12), (20, 12), seed=seed + 20)
    # patch 64, stride 32 and a 15 x 15 PSF
    random_case("tiledsv_p64_s32", 1, 1, 160, 144, 15, 15, 64, 32, use_fft=False, seed=seed + 30)
    # the reference's generator: one motion-blur PSF per patch
    gen = TiledBlurGenerator(MotionBlurGenerator((9, 9)), patch_size=(24, 20), stride=(12, 10))
    h = gen.step(batch_size=2, img_size=(70, 64), seed=5)["filters"]
    operator_case("tiledsv_generator", torch.rand(2, 1, 70, 64, generator=g(6)), h, (24, 20), (12, 10), seed=7)


def algo_fixtures():
    x = torch.rand(1, 1, 30, 28, generator=g(20))
    nr, nc = TiledSpaceVaryingBlur.num_filters((30, 28), 12, 6)
    h = torch.rand(1, 1, nr * nc, 5, 5, generator=g(22))
    h = h / h.sum(dim=(-2, -1), keepdim=True)
    phys = TiledSpaceVaryingBlur(filters=h, patch_size=12, stride=6)
    with torch.no_grad():
        y0 = phys.A(x)
        y = y0 + 0.01 * torch.randn(y0.shape, generator=g(23))
        z = torch.rand(x.shape, generator=g(24))
        prox = phys.prox_l2(z, y, 0.5)
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
    save("tiledsv_algo", x=x, h=h, y=y, z=z, gamma=np.float32(0.5), prox=prox, pgd=pgd, patch=np.int32((12, 12)),
         stride=np.int32((6, 6)), max_iter=np.int32(phys.max_iter), tol=np.float64(phys.tol))


if __name__ == "__main__":
    torch.set_num_threads(1)
    operator_fixtures()
    algo_fixtures()
