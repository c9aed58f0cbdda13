"""Generate the MATLAB-resize golden vectors (tests/golden/resize_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_resize.py

Every fixture holds the inputs and outputs of deepinv v0.4.1 on CPU in float32:
  - resize_f{factor}_{aa|noaa}_*: `DownsamplingMatlab` A, A_adjoint (the reference's autograd adjoint, on the (H_out f, W_out f)
    image), A_dagger, and the prox_l2 outcome (a value, or the error it raises);
  - resize_tiny_*: an image smaller than the band, where the reference's reflect padding raises;
  - resize_up2: `imresize_matlab(x, scale=2)` and `imresize_matlab(x, sizes=...)`;
  - resize_upsampling_*: `Upsampling` A / A_adjoint for three paddings and two filters, and the prox_l2 outcome;
  - resize_pgd: a short PGD super-resolution run (L2 data term, Tikhonov prior) on `DownsamplingMatlab`.
Error cases store the exception type as its index in ERRORS (-1: no error).
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
from deepinv.physics import DownsamplingMatlab, Upsampling  # noqa: E402
from deepinv.physics.functional import imresize_matlab  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError", "IndexError")


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)


def outcome(fn):
    """(value or zeros(0), error index)"""
    try:
        return fn(), -1
    except Exception as e:  # noqa: BLE001  (the reference's exception type is the datum)
        return torch.zeros(0), ERRORS.index(type(e).__name__)


def downsampling(name, factor, aa, shape, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    p = DownsamplingMatlab(factor=factor, antialiasing=aa)
    y = p.A(x)
    v = torch.randn(y.shape, generator=g)
    at = p.A_adjoint(v)
    z = torch.rand(at.shape, generator=g)
    dag = p.A_dagger(y)
    prox, prox_err = outcome(lambda: p.prox_l2(x, y, 0.5))
    prox_even = p.prox_l2(z, y, 0.5)
    save(name, x=x, y=y, v=v, At=at, dagger=dag, prox=prox, prox_err=prox_err, z=z, prox_even=prox_even, factor=factor,
         aa=int(aa), stored_factor=p.factor, max_iter=p.max_iter, tol=p.tol)


def main():
    downsampling("resize_f2_aa_odd", 2, True, (2, 3, 23, 17), 0)
    downsampling("resize_f3_aa_odd", 3, True, (2, 3, 23, 17), 1)
    downsampling("resize_f4_aa_odd", 4, True, (1, 2, 37, 29), 2)
    downsampling("resize_f2_noaa_odd", 2, False, (2, 1, 21, 30), 3)
    downsampling("resize_f4_noaa_odd", 4, False, (1, 3, 33, 19), 4)
    downsampling("resize_f3_aa_even", 3, True, (1, 1, 48, 36), 5)
    downsampling("resize_f15_aa", 1.5, True, (2, 2, 8, 9), 6)

    # images smaller than the band: the reference's reflect padding indexes past the axis
    for name, f, shape in (("resize_tiny_3x5_f4", 4, (1, 1, 3, 5)), ("resize_tiny_7x9_f4", 4, (2, 1, 7, 9)),
                           ("resize_tiny_9x3_f2", 2, (1, 1, 9, 3))):
        x = torch.rand(shape, generator=torch.Generator().manual_seed(7))
        y, err = outcome(lambda: DownsamplingMatlab(factor=f).A(x))
        save(name, x=x, y=y, err=err, factor=f)

    g = torch.Generator().manual_seed(8)
    x = torch.rand(2, 3, 11, 14, generator=g)
    save("resize_up2", x=x, up2=imresize_matlab(x, scale=2), up_sizes=imresize_matlab(x, sizes=(25, 17)),
         down_sizes=imresize_matlab(x, sizes=(6, 9)), up2_noaa=imresize_matlab(x, scale=2, antialiasing=False),
         x3=x[0], up2_3d=imresize_matlab(x[0], scale=2))

    for filt in ("bicubic", "gaussian"):
        for pad in ("circular", "reflect", "replicate"):
            g = torch.Generator().manual_seed(9)
            x = torch.rand(1, 3, 8, 8, generator=g)
            u = Upsampling(img_size=(3, 16, 16), filter=filt, factor=2, padding=pad)
            y = u.A(x)
            v = torch.randn(y.shape, generator=g)
            at = u.A_adjoint(v)
            prox, prox_err = outcome(lambda: u.prox_l2(x, v, 0.5))
            save(f"resize_upsampling_{filt}_{pad}", x=x, y=y, v=v, At=at, prox=prox, prox_err=prox_err,
                 filter=u.filter, max_iter=u.max_iter, tol=u.tol)
    _, err = outcome(lambda: Upsampling(img_size=(3, 16, 16), filter="bicubic", padding="valid"))
    save("resize_upsampling_valid", err=err)

    g = torch.Generator().manual_seed(10)
    x = torch.rand(1, 3, 32, 24, generator=g)
    p = DownsamplingMatlab(factor=2)
    y = p.A(x) + 0.01 * torch.randn(p.A(x).shape, generator=g)
    algo = PGD(data_fidelity=L2(), prior=Tikhonov(), stepsize=1.0, lambda_reg=0.1, max_iter=8, early_stop=False)
    with torch.no_grad():
        out = algo(y, p)
    save("resize_pgd", x=x, y=y, pgd=out, max_iter=8, stepsize=1.0, lambda_reg=0.1)


if __name__ == "__main__":
    main()
