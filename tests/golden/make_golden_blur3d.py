"""Generate the 3-D blur golden vectors (tests/golden/blur3d_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_blur3d.py

Every operator fixture stores the inputs and outputs of deepinv v0.4.1's `Blur` on (B, C, D, H, W) volumes, on CPU in float32:
x, k (the filter), v (a random point of A's range) and, per padding p, `A_<p>` = A x and `At_<p>` = A^T v (with `v_<p>` when A's
range differs from x's shape, i.e. valid), or `err_<p>` = the exception type the reference raised, as its index in ERRORS.  The adjointness
pair <A x, v> = <x, A^T v> is evaluated on these arrays by the tests.  `use_fft` records which convolution the reference ran.
`blur3d_algo` holds a CG `prox_l2` and a PGD run with Tikhonov on a 3-D circular blur, and a GD run with ZeroPrior.
"""
from __future__ import annotations

import warnings
from pathlib import Path

import numpy as np
import torch

warnings.filterwarnings("ignore")
import deepinv as dinv  # noqa: E402  (the real reference)
from deepinv.optim import GD, PGD  # noqa: E402
from deepinv.optim.data_fidelity import L2  # noqa: E402
from deepinv.optim.prior import Tikhonov, ZeroPrior  # noqa: E402
from deepinv.physics import Blur  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
PADS = ("valid", "circular", "replicate", "reflect", "constant")
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")  # the fixtures' `err_<p>` codes


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def operator_case(name, shape, fshape, pads=PADS, use_fft=False, seed=0):
    x = torch.randn(*shape, generator=g(seed))
    k = torch.randn(*fshape, generator=g(seed + 1))
    out = dict(x=x, k=k, use_fft=np.int32(use_fft))
    for pad in pads:
        phys = Blur(filter=k, padding=pad, use_fft=use_fft)
        try:
            with torch.no_grad():
                y = phys.A(x)
                v = torch.randn(y.shape, generator=g(seed + 2))
                at = phys.A_adjoint(v)
        except Exception as e:  # noqa: BLE001  (recorded: the drop-in must raise the same type)
            out[f"err_{pad}"] = np.int32(ERRORS.index(type(e).__name__))
            continue
        assert at.shape == x.shape, (name, pad, at.shape, x.shape)
        out[f"A_{pad}"], out[f"v_{pad}"], out[f"At_{pad}"] = y, v, at
    save(name, **out)


def operator_fixtures():
    # odd and even filters along each axis, a unit filter and a single-plane (1 x h x w) filter; all five paddings
    for tag, fs in (("3x3x3", (3, 3, 3)), ("4x5x2", (4, 5, 2)), ("5x3x4", (5, 3, 4)), ("1x1x1", (1, 1, 1)), ("1x5x5", (1, 5, 5)),
                    ("2x2x2", (2, 2, 2))):
        operator_case(f"blur3d_{tag}", (2, 2, 7, 9, 10), (1, 1, *fs), seed=sum(fs))
    # the four filter broadcasts
    for fn, (fb, fc) in {"11": (1, 1), "B1": (2, 1), "1C": (1, 3), "BC": (2, 3)}.items():
        operator_case(f"blur3d_bcast_f{fn}", (2, 3, 6, 8, 9), (fb, fc, 3, 4, 5), seed=40 + fb + fc)
    # volumes smaller than the filter in one axis (depth, rows, columns); reflect and valid then raise in the reference
    operator_case("blur3d_small_D", (1, 2, 2, 8, 9), (1, 1, 5, 3, 3), seed=50)
    operator_case("blur3d_small_H", (1, 1, 6, 3, 9), (1, 1, 3, 7, 3), seed=51)
    operator_case("blur3d_small_W", (2, 1, 6, 8, 2), (1, 1, 3, 3, 4), seed=52)
    # the FFT convolutions, odd filters (their centre is the direct one's)
    operator_case("blur3d_fft_3x5x3", (2, 1, 8, 10, 9), (1, 1, 3, 5, 3), use_fft=True, seed=60)
    operator_case("blur3d_fft_bcast", (2, 2, 6, 7, 8), (2, 2, 5, 3, 3), use_fft=True, seed=61)


def algo_fixtures():
    x = torch.rand(1, 1, 8, 12, 10, generator=g(70))
    k = torch.rand(1, 1, 3, 5, 5, generator=g(71))
    k = k / k.sum()
    phys = Blur(filter=k, padding="circular")
    with torch.no_grad():
        y0 = phys.A(x)
        y = y0 + 0.01 * torch.randn(y0.shape, generator=g(72))
        z = torch.rand(x.shape, generator=g(73))
        prox = phys.prox_l2(z, y, 0.5)
        pgd = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=6, early_stop=False)(y, phys)
        gd = GD(data_fidelity=L2(), prior=ZeroPrior(), stepsize=1.0, max_iter=6, early_stop=False)(y, phys)
    save("blur3d_algo", x=x, k=k, y=y, z=z, gamma=np.float32(0.5), prox=prox, pgd=pgd, gd=gd, max_iter=np.int32(phys.max_iter),
         tol=np.float64(phys.tol))


if __name__ == "__main__":
    torch.set_num_threads(1)
    operator_fixtures()
    algo_fixtures()
