"""TV prox denoisers on libdinvk (deepinv/models/tv.py): `TVDenoiser` and `TVL1Denoiser`.

Same constructor, attributes and `forward(y, ths)` as the reference, including its warm restart: the state (x2, u2) of
the last call is kept (detached) and starts the next call of the same shape.  The Chambolle-Pock loop runs in
`dinvk_tv_prox`, K iterations per launch, with the reference's break test evaluated on the device; the host reads the
solve's control block every `check_every` launches instead of once per iteration.  2-D only; not differentiable.
"""
from __future__ import annotations

import torch

from .. import ops
from .base import Denoiser


def _no_grad_guard_tv(name: str, *tensors) -> None:
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
        raise NotImplementedError(
            f"{name}: the TV prox kernel does not propagate gradients (the reference differentiates by unrolling its loop); "
            "call it under torch.no_grad() or on tensors that do not require grad."
        )


class TVDenoiser(Denoiser):
    """Proximal operator of the isotropic total variation, argmin_x 1/2 ||x - y||^2 + ths ||Dx||_{1,2}."""

    l1 = False

    def __init__(self, verbose: bool = False, tau: float = 0.01, rho: float = 1.99, n_it_max: int = 1000, crit: float = 1e-5,
                 x2: torch.Tensor = None, u2: torch.Tensor = None, ths: float | torch.Tensor = None, check_every: int = 16):
        super().__init__()
        self.verbose = verbose
        self.n_it_max = n_it_max
        self.crit = crit
        self.restart = True
        self.ths = ths
        self.tau = tau
        self.rho = rho
        self.x2 = x2
        self.u2 = u2
        self.has_converged = False
        self.check_every = check_every  # launches between two reads of the control block (each read synchronises)
        self.n_iter = None              # iterations run by the last call (0-d int32 device tensor)

    def forward(self, y: torch.Tensor, ths: float | torch.Tensor = None, **kwargs) -> torch.Tensor:
        if ths is None and self.ths is None:
            raise RuntimeError(
                "Regularization parameter (ths) was not passed at init nor at forward. Please provide ths to one of these methods."
            )
        elif ths is None:
            ths = self.ths
        if y.dim() != 4:
            raise NotImplementedError(f"{type(self).__name__}: only 2-D images (B, C, H, W) are supported, got {y.dim()}-D input "
                                      "(3-D total variation is not implemented)")
        _no_grad_guard_tv(type(self).__name__, y, ths)
        restart = self.restart or self.x2 is None or self.u2 is None or self.x2.shape != y.shape
        if restart:
            x2 = y
            u2 = torch.zeros((*y.shape, y.ndim - 2), device=y.device, dtype=y.dtype)
            self.restart = False
        else:
            x2, u2 = self.x2, self.u2
        if isinstance(ths, torch.Tensor):
            ths = ths.squeeze()
        lambd = self._handle_sigma(ths, batch_size=y.size(0), device=y.device, dtype=torch.float32)
        with torch.no_grad():
            x2, u2, self.n_iter = ops.tv_prox(y, lambd.reshape(-1), x2, u2, l1=self.l1, tau=self.tau, rho=self.rho,
                                               n_it_max=self.n_it_max, crit=self.crit, check_every=self.check_every)
        if self.verbose and self.n_iter is not None and int(self.n_iter) < self.n_it_max:
            print("TV prox reached convergence")
        x2 = x2.to(y.dtype)
        self.x2 = x2.detach()
        self.u2 = u2.to(y.dtype).detach()
        return x2

    @staticmethod
    def nabla(x: torch.Tensor) -> torch.Tensor:
        if x.ndim not in [4, 5]:
            raise ValueError(f"Input tensor must be 4D or 5D, got {x.ndim}D")
        return ops.tv_nabla(x)

    @staticmethod
    def nabla_adjoint(x: torch.Tensor) -> torch.Tensor:
        if x.ndim not in [5, 6]:
            raise ValueError(f"Input tensor must be 5D or 6D, got {x.ndim}D")
        return ops.tv_nabla_adjoint(x)


class TVL1Denoiser(TVDenoiser):
    """TV-L1 variant: the dual step clamps each difference to [-ths, ths] (tv.py:221-239)."""

    l1 = True
