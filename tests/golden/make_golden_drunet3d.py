"""Generate the 3-D DRUNet golden vectors (tests/golden/drunet3d_*.npz) by running the REAL reference.

Run in the authoring container only, like make_golden.py:

    PYTHONPATH=oracle/_shim:/root/reference python tests/golden/make_golden_drunet3d.py

Every fixture holds the inputs and outputs of deepinv v0.4.1's `DRUNet(dim=3)` on CPU in float32, at small widths
(nc = (64, 64, 128, 128), nb = 1).  The weights are not stored: `weights(seed, sd)` regenerates them from a seed with torch's CPU
generator, and the fixture stores `wsum` = (sum, sum of squares, first value) of the regenerated tensors, so that a torch version
whose generator draws differently fails loudly instead of comparing against the wrong network.  `keys` / `shapes` are the
reference's 3-D state_dict names and shapes.  Error cases store the exception type as its index in ERRORS.
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
from deepinv.optim.prior import PnP  # noqa: E402
from deepinv.physics import MRI, Blur  # noqa: E402

OUT = Path(__file__).resolve().parent
assert dinv.__version__ == "0.4.1", dinv.__version__
ERRORS = ("RuntimeError", "ValueError", "AssertionError", "NotImplementedError")
NC, NB = (64, 64, 128, 128), 1


def weights(seed, shapes):
    """deterministic weights for the state_dict names / shapes `shapes` (dict), scaled like the reference's orthogonal init"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        s = tuple(shapes[k])
        fan = int(np.prod(s[1:]))
        out[k] = torch.randn(s, generator=g) * (0.5 / fan ** 0.5)
    return out


def wsum(sd):
    ks = sorted(sd)
    return np.array([sum(float(sd[k].double().sum()) for k in ks), sum(float(sd[k].double().pow(2).sum()) for k in ks),
                     float(sd[ks[0]].reshape(-1)[0])])


def model(ch, seed):
    m = dinv.models.DRUNet(in_channels=ch, out_channels=ch, nc=NC, nb=NB, pretrained=None, dim=3).eval()
    sd = weights(seed, {k: v.shape for k, v in m.state_dict().items()})
    m.load_state_dict(sd, strict=True)
    return m, sd


def save(name, **arrays):
    conv = {k: np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrays.items()}
    np.savez_compressed(OUT / f"{name}.npz", **conv)
    print(f"{name}: {len(conv)} arrays, {sum(v.nbytes for v in conv.values()) / 1024:.0f} KiB")


def g(seed):
    return torch.Generator().manual_seed(seed)


def sd_arrays(sd, seed):
    keys = sorted(sd)
    shapes = np.zeros((len(keys), 5), dtype=np.int32)
    for i, k in enumerate(keys):
        shapes[i, : sd[k].dim()] = sd[k].shape
    return dict(seed=np.int32(seed), wsum=wsum(sd), keys=np.array(keys), shapes=shapes)


def err_index(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return np.int32(ERRORS.index(type(e).__name__))
    raise AssertionError("the reference used to raise here")


def main():
    with torch.no_grad():
        # a safe shape, C = 2, scalar and (B, 1, 1, 1, 1) sigma
        m, sd = model(2, 100)
        x = torch.randn(1, 2, 32, 32, 40, generator=g(1))
        save("drunet3d_safe", x=x, sigma=np.float32(0.05), out=m(x, 0.05), sigma5=torch.full((1, 1, 1, 1, 1), 0.08),
             out5=m(x, torch.full((1, 1, 1, 1, 1), 0.08)), **sd_arrays(sd, 100),
             err_sigma4=err_index(lambda: m(x, torch.ones(1, 1, 1, 1))),
             err_onesplit=err_index(lambda: m(torch.zeros(1, 2, 64, 70, 66), 0.05)),
             err_dim=err_index(lambda: dinv.models.DRUNet(pretrained=None, dim=4)))
        # padded shapes: C = 1 with (B,) sigma; C = 2 with a full noise map
        m1, sd1 = model(1, 200)
        x = torch.randn(2, 1, 16, 24, 20, generator=g(2))
        s = torch.tensor([0.03, 0.09])
        save("drunet3d_pad_c1", x=x, sigma=s, out=m1(x, s), **sd_arrays(sd1, 200))
        x = torch.randn(2, 2, 8, 16, 16, generator=g(3))
        s = 0.1 * torch.rand(2, 1, 8, 16, 16, generator=g(4))
        save("drunet3d_pad_map", x=x, sigma=s, out=m(x, s), **sd_arrays(sd, 100))
        # PnP-PGD on 3-D single-coil MRI and on a 3-D circular Blur
        D, H, W = 8, 16, 16
        x = torch.randn(1, 2, D, H, W, generator=g(5))
        mask = (torch.rand(D, H, W, generator=g(6)) > 0.5).float()
        phys = MRI(mask=mask, img_size=(2, D, H, W), three_d=True)
        y = phys.A(x)
        out = PGD(data_fidelity=L2(), prior=PnP(m), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)(y, phys)
        save("drunet3d_pgd_mri", x=x, mask=mask, y=y, out=out, **sd_arrays(sd, 100))
        x = torch.rand(1, 1, D, H, W, generator=g(7))
        filt = torch.rand(1, 1, 3, 3, 3, generator=g(8))
        filt = filt / filt.sum()
        phys = Blur(filter=filt, padding="circular")
        y = phys.A(x)
        out = PGD(data_fidelity=L2(), prior=PnP(m1), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)(y, phys)
        save("drunet3d_pgd_blur", x=x, filt=filt, y=y, out=out, **sd_arrays(sd1, 200))


if __name__ == "__main__":
    main()
