"""Generate the 3-D MRI golden vectors (tests/golden/mri3d_*.npz, except mri3d_6x8x12 which make_golden.py writes) by running the
REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_mri3d.py

Every fixture stores the inputs and outputs of deepinv v0.4.1's `MRI(three_d=True)` / `MultiCoilMRI(three_d=True)` on CPU in
float32.  Multi-coil fixtures: x (B,2,D,H,W), mask_in (what the constructor was given), maps_re / maps_im (B|1,N,D,H,W), y = A x,
At = A^T y, At_crop = A^T(y, crop=True), z / gamma and prox = the CG prox_l2, dagger = the CG A_dagger (SENSE), with the solver's
max_iter / tol, and err_rss = the exception type `A_adjoint(rss=True)` raised, as its index in ERRORS.  Single-coil fixtures: x,
mask_in, y, At, AtA, z / gamma / prox, dagger and err_mag = the exception type `A_adjoint(mag=True)` raised.
`mri3d_mc_pgd` holds a PGD run with L2 + Tikhonov.
"""
from __future__ import annotations

import warnings
from math import sqrt
from pathlib import Path

import numpy as np
import torch

warnings.filterwarnings("ignore")
import deepinv as dinv  # noqa: E402  (the real reference)
from deepinv.optim import PGD  # noqa: E402
from deepinv.optim.data_fidelity import L2  # noqa: E402
from deepinv.optim.prior import Tikhonov  # noqa: E402
from deepinv.physics import MRI, MultiCoilMRI  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")
MAX_ITER, TOL = 30, 1e-6


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def multicoil_case(name, B, N, dims, mask_in, maps, seed):
    img = (2, *dims)
    phys = MultiCoilMRI(mask=mask_in, coil_maps=maps, img_size=img, three_d=True)
    phys.max_iter, phys.tol = MAX_ITER, TOL
    x = torch.randn(B, *img, generator=g(seed))
    z = torch.randn(B, *img, generator=g(seed + 1))
    gamma = 0.8
    out = dict(x=x, mask_in=mask_in, maps_re=maps.real, maps_im=maps.imag, z=z, gamma=np.float32(gamma),
               max_iter=np.int32(MAX_ITER), tol=np.float32(TOL))
    with torch.no_grad():
        y = phys.A(x)
        out.update(mask=phys.mask, y=y, At=phys.A_adjoint(y), At_crop=phys.A_adjoint(y, crop=True))
        try:
            phys.A_adjoint(y, rss=True)
            raise AssertionError("the reference's 3-D rss used to raise")
        except (ValueError, RuntimeError) as e:
            out["err_rss"] = np.int32(ERRORS.index(type(e).__name__))
        out["dagger"] = phys.A_dagger(y)
        out["prox"] = phys.prox_l2(z, y, gamma)
    save(name, **out)


def singlecoil_case(name, B, dims, mask_in, seed):
    img = (2, *dims)
    phys = MRI(mask=mask_in, img_size=img, three_d=True)
    x = torch.randn(B, *img, generator=g(seed))
    z = torch.randn(B, *img, generator=g(seed + 1))
    gamma = 0.6
    with torch.no_grad():
        y = phys.A(x)
        out = dict(x=x, mask_in=mask_in, mask=phys.mask, y=y, At=phys.A_adjoint(y), AtA=phys.A_adjoint_A(x), z=z,
                   gamma=np.float32(gamma), prox=phys.prox_l2(z, y, gamma), dagger=phys.A_dagger(y))
        try:
            phys.A_adjoint(y, mag=True)
            raise AssertionError("the reference's 3-D mag used to raise")
        except (ValueError, RuntimeError) as e:
            out["err_mag"] = np.int32(ERRORS.index(type(e).__name__))
    save(name, **out)


def cmaps(b, N, dims, seed):
    m = torch.randn(b, N, *dims, generator=g(seed), dtype=torch.complex64)
    return m / m.abs().pow(2).sum(1, keepdim=True).sqrt()


def main():
    # the reference's own test operators (deepinv/tests/test_physics.py:184-188, 218-231): (2,5,17,11), 15 coils of ones / sqrt(15)
    dims = (5, 17, 11)
    ones = torch.ones(1, 15, *dims, dtype=torch.complex64) / sqrt(15)
    multicoil_case("mri3d_mc_reference_op", 2, 15, dims, torch.ones(*dims), ones, 10)
    singlecoil_case("mri3d_sc_reference_op", 2, dims, torch.ones(*dims), 20)
    # per-batch maps and masks; shared maps and mask; a single coil; prime sizes (O(N²) path) and powers of two
    multicoil_case("mri3d_mc_per_batch", 2, 4, (6, 10, 12), (torch.rand(2, 1, 6, 10, 12, generator=g(31)) > 0.4).float(),
                   cmaps(2, 4, (6, 10, 12), 32), 30)
    multicoil_case("mri3d_mc_shared_prime", 3, 3, (7, 13, 11), (torch.rand(7, 13, 11, generator=g(41)) > 0.5).float(),
                   cmaps(1, 3, (7, 13, 11), 42), 40)
    multicoil_case("mri3d_mc_one_coil", 2, 1, (8, 16, 16), (torch.rand(8, 16, 16, generator=g(51)) > 0.5).float(),
                   cmaps(1, 1, (8, 16, 16), 52), 50)
    singlecoil_case("mri3d_sc_pow2", 2, (8, 16, 16), (torch.rand(2, 8, 16, 16, generator=g(61)) > 0.5).float().unsqueeze(1), 60)
    singlecoil_case("mri3d_sc_prime", 1, (5, 7, 13), (torch.rand(5, 7, 13, generator=g(71)) > 0.5).float(), 70)

    # a short PGD run with L2 + Tikhonov on 3-D multi-coil
    dims = (6, 12, 10)
    maps = cmaps(1, 4, dims, 81)
    phys = MultiCoilMRI(mask=(torch.rand(*dims, generator=g(82)) > 0.4).float(), coil_maps=maps, img_size=(2, *dims), three_d=True)
    x = torch.randn(1, 2, *dims, generator=g(83))
    with torch.no_grad():
        y = phys.A(x) + 0.01 * phys.mask[:, :, None] * torch.randn(1, 2, 4, *dims, generator=g(84))
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=8, early_stop=False)(y, phys)
    save("mri3d_mc_pgd", x=x, mask=phys.mask, maps_re=maps.real, maps_im=maps.imag, y=y, pgd=pgd)


if __name__ == "__main__":
    main()
