"""Cartesian MRI mask generators, sampled ON the device for the whole batch at once (SURVEY §8(f) item 4;
deepinv/physics/generator/mri.py:15-389, generator/base.py:20-183).

Same classes, constructor arguments, `step(batch_size, seed, img_size)` contract and output shapes/values
((B,C,H,W) or (B,C,T,H,W), entries in {0,1}, lines constant along H) as the reference, so the result can be handed to
`MRI(mask=...)` / `physics.update(mask=...)` without leaving the GPU.  The reference draws the lines of every (sample,
frame) in a Python double loop of `multinomial(..., replacement=False)` calls; here ONE batched draw does it: sampling k
columns without replacement with probabilities ∝ pdf is the Plackett-Luce law, which is exactly the law of the top-k
of `log pdf + Gumbel noise` — a (B*T, W) noise tensor and one `topk`.  The distribution is the reference's; the random
stream is not (torch's sampler consumes its generator differently), so parity is on the law — line counts, fixed centre
band, inclusion frequencies measured on the real reference (tests/golden/maskgen_stats.npz) — not draw by draw.
"""
from __future__ import annotations

import warnings

import torch
import torch.nn as nn


class PhysicsGenerator(nn.Module):
    """parameter generator base (generator/base.py:20-183): holds the device / dtype and a torch.Generator"""

    def __init__(self, step=lambda **kwargs: {}, rng: torch.Generator | None = None, device="cpu", dtype=torch.float32, **kwargs):
        super().__init__()
        self.step_func = step
        self.kwargs = kwargs
        self.factory_kwargs = {"device": device, "dtype": dtype}
        self.device = torch.device(device)
        if rng is None:
            self.rng = torch.Generator(device=device)
        else:
            if rng.device != self.device:
                raise RuntimeError(f"The random generator is not on the same device as the Physics Generator. "
                                   f"Got random generator on {rng.device} and the Physics Generator on {self.device}.")
            self.rng = rng
        self.initial_random_state = self.rng.get_state()

    def step(self, batch_size: int = 1, seed: int | None = None, **kwargs) -> dict:
        self.rng_manual_seed(seed)
        if not kwargs:
            self.kwargs = kwargs
        return self.step_func(batch_size, seed, **kwargs)

    def rng_manual_seed(self, seed: int | None = None):
        if seed is not None:
            self.rng = self.rng.manual_seed(seed)

    def reset_rng(self):
        self.rng.set_state(self.initial_random_state)


class BaseMaskGenerator(PhysicsGenerator):
    """vertical-line masks: a fully sampled centre band + `n_lines` further columns chosen by the child class"""

    def __init__(self, img_size: tuple, acceleration: int = 4, center_fraction: float | None = None,
                 rng: torch.Generator | None = None, device="cpu", *args, **kwargs):
        super().__init__(*args, **kwargs, rng=rng, device=device)
        self.img_size = img_size
        self.acc = acceleration
        self.center_fraction = center_fraction if center_fraction is not None else (0.08 if acceleration < 8 else 0.04)
        if len(img_size) == 2:
            (self.H, self.W), self.C, self.T = img_size, 1, 0
        elif len(img_size) == 3:
            (self.C, self.H, self.W), self.T = img_size, 0
        elif len(img_size) == 4:
            self.C, self.T, self.H, self.W = img_size
        else:
            raise ValueError("img_size must be (H, W) or (C, H, W) or (C, T, H, W)")
        self.calculate_lines(self.W)

    def calculate_lines(self, W: int):
        self.n_center = int(self.center_fraction * W)
        self.n_lines = int(W // self.acc - self.n_center)
        if self.n_lines < 0:
            raise ValueError("center_fraction is too high for this acceleration factor.")
        if self.n_lines == 0:
            warnings.warn("Number of high frequency lines to be sampled is 0. Reduce acceleration factor or reduce center_fraction.")

    def _center(self, W: int):
        return W // 2 - self.n_center // 2, W // 2 + -(-self.n_center // 2)

    def sample_columns(self, rows: int, frames: int, W: int) -> torch.Tensor:
        """(rows, frames, W) column indicator in {0,1} — the child class's sampling law"""
        raise NotImplementedError

    def step(self, batch_size: int = 1, seed: int | None = None, img_size: tuple | None = None, **kwargs) -> dict:
        self.rng_manual_seed(seed)
        B = 1 if batch_size == 0 else batch_size
        T = self.T if self.T > 0 else 1
        H, W = (self.H, self.W) if img_size is None else img_size
        self.calculate_lines(W)
        if self.n_lines + self.n_center >= W:
            cols = torch.ones(B, T, W, **self.factory_kwargs)
        else:
            cols = self.sample_columns(B, T, W).to(self.factory_kwargs["dtype"])
        mask = cols[:, None, :, None, :].expand(B, self.C, T, H, W).contiguous()
        if self.T == 0:
            mask = mask[:, :, 0]
        if batch_size == 0:
            mask = mask[0]
        return {"mask": mask}


class RandomMaskGenerator(BaseMaskGenerator):
    """uniformly random high-frequency columns (generator/mri.py:136-196)"""

    def get_pdf(self, W: int) -> torch.Tensor:
        return torch.ones(W, device=self.device)

    def sample_columns(self, rows: int, frames: int, W: int) -> torch.Tensor:
        lo, hi = self._center(W)
        pdf = self.get_pdf(W).clone()
        pdf[lo:hi] = 0  # the centre band is never drawn, it is always on
        cols = torch.zeros(rows * frames, W, device=self.device)
        if self.n_lines > 0:
            u = torch.rand(rows * frames, W, device=self.device, generator=self.rng).clamp_(1e-20, 1.0)
            keys = torch.log(pdf)[None] - torch.log(-torch.log(u))  # Gumbel top-k == sampling without replacement ∝ pdf
            idx = torch.topk(keys, self.n_lines, dim=1).indices
            cols.scatter_(1, idx, 1.0)
        cols[:, lo:hi] = 1
        return cols.reshape(rows, frames, W)


class GaussianMaskGenerator(RandomMaskGenerator):
    """tail-adjusted Gaussian density over the columns (generator/mri.py:284-324)"""

    def get_pdf(self, W: int) -> torch.Tensor:
        x = torch.arange(W, device=self.device)
        pdf = torch.exp(-(0.5 / (W / 10.0) ** 2) * (x - W / 2) ** 2)
        return pdf + (W / (2.0 * self.acc) * 1.0 / W)


class EquispacedMaskGenerator(BaseMaskGenerator):
    """equispaced columns with a random per-sample offset, sheared across time (generator/mri.py:327-389, after fastMRI)"""

    def sample_columns(self, rows: int, frames: int, W: int) -> torch.Tensor:
        pad = (W - self.n_center + 1) // 2
        adjusted = (self.acc * (self.n_center - W)) / (self.n_center * self.acc - W)
        offset = torch.randint(low=0, high=round(adjusted), size=(rows,), device=self.device, generator=self.rng)
        # column j of the n-th sample of (row b, frame t): round(((t + offset_b) mod adjusted) + n * adjusted), while < W - 1
        start = torch.remainder(torch.arange(frames, device=self.device)[None, :] + offset[:, None], adjusted)  # (rows, frames)
        nmax = int((W - 1) / adjusted) + 2
        pos = start[..., None] + torch.arange(nmax, device=self.device) * adjusted
        valid = pos < (W - 1)
        idx = torch.where(valid, pos.round().to(torch.int64), torch.full_like(pos, W, dtype=torch.int64))
        cols = torch.zeros(rows, frames, W + 1, device=self.device)
        cols.scatter_(2, idx, 1.0)
        cols = cols[..., :W]
        cols[..., pad: pad + self.n_center] = 1
        return cols


class PSFGenerator(PhysicsGenerator):
    """base class of PSF generators (generator/blur.py:16-60): holds `psf_size`"""

    def __init__(self, psf_size: tuple = (31, 31), num_channels: int = 1, **kwargs):
        extra = {k: kwargs.pop(k) for k in list(kwargs) if k not in ("rng", "device", "dtype", "step")}
        super().__init__(**kwargs)
        self.psf_size = psf_size
        self.num_channels = num_channels
        for k, v in extra.items():
            setattr(self, k, v)


class MotionBlurGenerator(PSFGenerator):
    r"""Random motion-blur PSFs (generator/blur.py:209-352, after Schuler et al. 2015): x(t), y(t) ~ GP(0, Matern-5/2-type
    kernel k), sampled by circulant embedding (irfft(rfft(noise) * sqrt(rfft(k)))) and rasterised as a 2-D histogram of the
    mean-free trajectory on [-1,1]^2, normalised to sum 1.  Same random draws as the reference (two `randn(B, n_steps)` from
    the generator), so a CPU generator with the same seed gives the reference's PSFs exactly; the per-trajectory Python loop of
    `histogramdd` calls is ONE batched `scatter_add` here, so a whole batch of PSFs is produced on the device in a few launches."""

    def __init__(self, psf_size: tuple, rng: torch.Generator | None = None, device="cpu", dtype=torch.float32, l: float = 0.3,
                 sigma: float = 0.25, n_steps: int = 1000):
        if isinstance(psf_size, int):
            psf_size = (psf_size, psf_size)
        if len(psf_size) != 2:
            raise ValueError("psf_size must 2D.")
        super().__init__(psf_size=psf_size, device=device, dtype=dtype, rng=rng, l=l, sigma=sigma, n_steps=n_steps)

    def matern_kernel(self, diff, sigma: float | None = None, l: float | None = None):
        sigma = self.sigma if sigma is None else sigma
        l = self.l if l is None else l
        fraction = 5 ** 0.5 * diff.abs() / l
        return sigma ** 2 * (1 + fraction + fraction ** 2 / 3) * torch.exp(-fraction)

    def f_matern(self, batch_size: int = 1, sigma: float | None = None, l: float | None = None):
        vec = torch.randn(batch_size, self.n_steps, generator=self.rng, **self.factory_kwargs)
        time = torch.linspace(-torch.pi, torch.pi, self.n_steps, **self.factory_kwargs)[None]
        kernel_fft = torch.fft.rfft(self.matern_kernel(time, sigma, l))
        traj = torch.fft.irfft(torch.fft.rfft(vec) * torch.sqrt(kernel_fft)).real
        keep = int(self.n_steps // (2 * torch.pi))
        return traj[:, :keep]

    def step(self, batch_size: int = 1, sigma: float | None = None, l: float | None = None, seed: int | None = None, **kwargs):
        self.rng_manual_seed(seed)
        fx = self.f_matern(batch_size, sigma, l)
        fy = self.f_matern(batch_size, sigma, l)
        pts = torch.stack([fx - fx.mean(1, keepdim=True), fy - fy.mean(1, keepdim=True)], dim=-1)  # (B, n, 2)
        h, w = self.psf_size
        bins = torch.tensor([h, w], device=pts.device)
        inside = ((pts >= -1) & (pts <= 1)).all(-1)
        idx = (bins * ((pts + 1) / 2)).long()
        idx = torch.minimum(idx, bins - 1).clamp_min_(0)  # the last bin includes the upper bound
        flat = idx[..., 0] * w + idx[..., 1]
        hist = torch.zeros(batch_size, h * w, **self.factory_kwargs)
        hist.scatter_add_(1, flat, inside.to(hist.dtype))
        kernel = hist.reshape(batch_size, 1, h, w)
        kernel = kernel / (kernel.sum(dim=(-2, -1), keepdim=True) + 1e-6)
        return {"filter": kernel}


class TiledBlurGenerator(PSFGenerator):
    r"""Filters of TiledSpaceVaryingBlur (generator/blur.py:1737-1799): one PSF of `psf_generator` per patch of the image.
    `step(batch_size, img_size, seed)` draws batch_size * K PSFs in one call of `psf_generator` and returns
    ``{"filters": (B, C, K, h, w)}`` with the reference's reshape, so a CPU generator with the same seed gives its filters."""

    def __init__(self, psf_generator: PSFGenerator, patch_size, stride=None, rng: torch.Generator | None = None, device="cpu",
                 **kwargs):
        from .functional import _resolve_tiling_params

        super().__init__(psf_size=psf_generator.psf_size, rng=rng, device=device, **kwargs)
        self.patch_size, self.stride = _resolve_tiling_params(patch_size, stride)
        self.pad_if_needed = True
        self.psf_generator = psf_generator

    def get_num_patches(self, img_size) -> tuple[int, int]:
        from .functional import _as_pair, _num_patches

        return _num_patches(_as_pair(img_size), self.patch_size, self.stride)

    def step(self, batch_size: int = 1, img_size=None, seed: int | None = None, **kwargs) -> dict:
        nr, nc = self.get_num_patches(img_size)
        psf = self.psf_generator.step(batch_size=batch_size * nr * nc, seed=seed, **kwargs)["filter"]
        return {"filters": psf.view(batch_size, nr * nc, -1, *self.psf_size).transpose(1, 2)}
