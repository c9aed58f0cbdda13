"""Generate the total-variation golden vectors (tests/golden/tv_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_tv.py

Every fixture stores its inputs next to the outputs of deepinv v0.4.1's `TVDenoiser`, `TVL1Denoiser`, `TVPrior`,
`TVL1Prior`, and PGD / PDCP with `TVPrior`, all on CPU in float32.  The reference does not return its iteration count;
`n_iter` is counted from its calls to torch.linalg.norm (two per iteration, tv.py:139-141).
"""
from __future__ import annotations

import warnings
from pathlib import Path

import numpy as np
import torch

warnings.filterwarnings("ignore")
import deepinv as dinv  # noqa: E402  (the real reference)
from deepinv.models import TVDenoiser, TVL1Denoiser  # noqa: E402
from deepinv.optim import PDCP, PGD  # noqa: E402
from deepinv.optim.data_fidelity import L2  # noqa: E402
from deepinv.optim.prior import TVL1Prior, TVPrior  # noqa: E402
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
        # name, class, shape, ths (float or per-sample list), n_it_max, crit
        ("tv_iso_c1", TVDenoiser, (2, 1, 23, 17), 0.1, 60, 0.0),
        ("tv_iso_c2_persample", TVDenoiser, (3, 2, 19, 29), [0.05, 0.2, 0.5], 50, 0.0),
        ("tv_iso_c3_early", TVDenoiser, (1, 3, 31, 21), 0.15, 300, 1e-3),
        ("tv_l1_c1", TVL1Denoiser, (2, 1, 21, 25), 0.1, 60, 0.0),
        ("tv_l1_c3_persample", TVL1Denoiser, (2, 3, 17, 15), [0.03, 0.3], 40, 0.0),
        ("tv_iso_ths0", TVDenoiser, (2, 2, 13, 11), 0.0, 30, 0.0),
    ]
    for name, cls, shape, ths, n_it, crit in cases:
        y = image(*shape, seed=len(name))
        y2 = image(*shape, seed=len(name) + 100)
        ths_t = torch.tensor(ths, dtype=torch.float32) if isinstance(ths, list) else torch.tensor(float(ths))
        den = cls(n_it_max=n_it, crit=crit)
        with torch.no_grad(), count_iterations() as c1:
            out1 = den(y, ths=ths if not isinstance(ths, list) else ths_t)
        x2_1, u2_1 = den.x2.clone(), den.u2.clone()
        with torch.no_grad(), count_iterations() as c2:
            out2 = den(y2, ths=ths if not isinstance(ths, list) else ths_t)  # warm restart from (x2_1, u2_1)
        save(name, y=y, y2=y2, ths=ths_t, l1=np.int32(cls is TVL1Denoiser), n_it_max=np.int32(n_it), crit=np.float64(crit),
             out1=out1, x2_1=x2_1, u2_1=u2_1, n_iter1=np.int32(c1.iters), out2=out2, u2_2=den.u2, n_iter2=np.int32(c2.iters))


def prior_fixtures():
    x = image(2, 3, 14, 19, seed=7)
    x[..., :4, :5] = 0.25  # a flat patch: the subgradient takes the zero element there
    gfield = torch.randn(2, 3, 14, 19, 2, generator=g(8))
    p, p1 = TVPrior(), TVL1Prior()
    save("tv_prior", x=x, gfield=gfield, fn=p.fn(x), fn_l1=p1.fn(x), grad=p.grad(x), nabla=p.nabla(x),
         nabla_adjoint=p.nabla_adjoint(gfield))


def algo_fixtures():
    # the reference's test_priors_algo setting in miniature: circular Blur, TVPrior, PGD and PDCP
    x = image(1, 1, 24, 20, seed=9).clamp(0, 1.5)
    filt = torch.ones(1, 1, 3, 3) / 9.0
    phys = Blur(filter=filt, padding="circular")
    y = phys.A(x) + 0.01 * torch.randn(x.shape, generator=g(10))
    with torch.no_grad():
        pgd = PGD(data_fidelity=L2(), prior=TVPrior(n_it_max=200), stepsize=1.0, lambda_reg=0.05, max_iter=5, early_stop=False)(y, phys)
        pdcp = PDCP(data_fidelity=L2(), prior=TVPrior(n_it_max=200), lambda_reg=0.05, stepsize=0.5, stepsize_dual=0.5, max_iter=5,
                    early_stop=False)(y, phys)
    save("tv_algo_blur", x=x, filt=filt, y=y, pgd=pgd, pdcp=pdcp)


if __name__ == "__main__":
    torch.set_num_threads(1)
    denoiser_fixtures()
    prior_fixtures()
    algo_fixtures()
