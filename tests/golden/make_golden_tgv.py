"""Generate the total-generalized-variation golden vectors (tests/golden/tgv_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden_tv.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_tgv.py

Every fixture stores its inputs next to the outputs of deepinv v0.4.1's `TGVDenoiser` (two calls: a restart and a warm
restart from the first call's state), its `epsilon` / `epsilon_adjoint`, and PGD with `PnP(TGVDenoiser(...))`, all on
CPU in float32.  The reference does not return its iteration count; `n_iter` is counted from its calls to
torch.linalg.norm (two per iteration with verbose=False, tgv.py:162-164).
"""
from __future__ import annotations

import warnings
from pathlib import Path

import numpy as np
import torch

warnings.filterwarnings("ignore")
import deepinv as dinv  # noqa: E402  (the real reference)
from deepinv.models import TGVDenoiser  # noqa: E402
from deepinv.optim import PGD  # noqa: E402
from deepinv.optim.data_fidelity import L2  # noqa: E402
from deepinv.optim.prior import PnP  # noqa: E402
from deepinv.physics import Blur  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def image(B, C, H, W, seed):
    """a smooth ramp plus noise: no two neighbouring pixels are equal, so no difference vanishes"""
    base = torch.linspace(0, 1, W).expand(H, W) + torch.linspace(0, 0.5, H)[:, None]
    return (base + 0.3 * torch.randn(B, C, H, W, generator=g(seed))).float()


class count_iterations:
    def __enter__(self):
        self.n, self._norm = 0, torch.linalg.norm

        def norm(*a, **k):
            self.n += 1
            return self._norm(*a, **k)

        torch.linalg.norm = norm
        return self

    def __exit__(self, *exc):
        torch.linalg.norm = self._norm

    @property
    def iters(self):
        return self.n // 2


def denoiser_fixtures():
    cases = [
        # name, shape, ths (float or per-sample list), n_it_max, crit
        ("tgv_c1", (2, 1, 61, 53), 0.1, 40, 0.0),
        ("tgv_c3", (1, 3, 53, 67), 0.2, 30, 0.0),
        ("tgv_persample", (3, 2, 29, 51), [0.05, 0.2, 0.5], 30, 0.0),
        ("tgv_early", (1, 2, 57, 50), 1.0, 400, 2.98e-3),  # breaks at iteration 78: inside a launch of 2 or 4
        ("tgv_ths0", (2, 1, 13, 11), 0.0, 8, 0.0),
    ]
    for name, shape, ths, n_it, crit in cases:
        y = image(*shape, seed=len(name))
        y2 = image(*shape, seed=len(name) + 100)
        ths_t = torch.tensor(ths, dtype=torch.float32) if isinstance(ths, list) else torch.tensor(float(ths))
        den = TGVDenoiser(n_it_max=n_it, crit=crit)
        with torch.no_grad(), count_iterations() as c1:
            out1 = den(y, ths=ths if not isinstance(ths, list) else ths_t).clone()
        x2_1, r2_1, u2_1 = den.x2.clone(), den.r2.clone(), den.u2.clone()
        conv1 = den.has_converged
        with torch.no_grad(), count_iterations() as c2:
            out2 = den(y2, ths=ths if not isinstance(ths, list) else ths_t).clone()  # warm restart from the first call's state
        save(name, y=y, y2=y2, ths=ths_t, n_it_max=np.int32(n_it), crit=np.float64(crit), out1=out1, x2_1=x2_1, r2_1=r2_1,
             u2_1=u2_1, n_iter1=np.int32(c1.iters), converged1=np.int32(conv1), out2=out2, r2_2=den.r2, u2_2=den.u2,
             n_iter2=np.int32(c2.iters), converged2=np.int32(den.has_converged))


def stencil_fixtures():
    f = torch.randn(2, 3, 14, 19, 2, generator=g(21))
    gf = torch.randn(2, 3, 14, 19, 4, generator=g(22))
    save("tgv_stencils", f=f, gfield=gf, epsilon=TGVDenoiser.epsilon(f), epsilon_adjoint=TGVDenoiser.epsilon_adjoint(gf))


def algo_fixtures():
    # PnP-PGD with the TGV prox as the denoiser on circular Blur (the reference's test_optim setting in miniature)
    x = image(1, 1, 24, 20, seed=9).clamp(0, 1.5)
    filt = torch.ones(1, 1, 3, 3) / 9.0
    phys = Blur(filter=filt, padding="circular")
    y = phys.A(x) + 0.01 * torch.randn(x.shape, generator=g(10))
    with torch.no_grad():
        pgd = PGD(data_fidelity=L2(), prior=PnP(TGVDenoiser(n_it_max=100, crit=1e-5)), stepsize=1.0, sigma_denoiser=0.05,
                  max_iter=5, early_stop=False)(y, phys)
    save("tgv_algo_blur", x=x, filt=filt, y=y, pgd=pgd)


if __name__ == "__main__":
    torch.set_num_threads(1)
    denoiser_fixtures()
    stencil_fixtures()
    algo_fixtures()
