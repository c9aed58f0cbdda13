"""TGV prox denoiser on libdinvk (deepinv/models/tgv.py): `TGVDenoiser`.

Same constructor, attributes and `forward(y, ths)` as the reference, including its warm restart: the state (x2, r2, u2)
of the last call is kept (detached) and starts the next call of the same shape, and `has_converged` is set once the
break test passes.  The over-relaxed Chambolle-Pock loop runs in `dinvk_tgv_prox`, K iterations per launch, with the
reference's break test evaluated on the device; the host reads the solve's control block every `check_every` launches
instead of once per iteration.  2-D only; not differentiable.  `verbose` prints the reference's convergence and
non-convergence messages but not its primal-cost line every 100 iterations (that would need the iterate on the host).
"""
from __future__ import annotations

import torch

from .. import ops
from .base import Denoiser
from .tv import TVDenoiser, _no_grad_guard_tv


class TGVDenoiser(Denoiser):
    """Proximal operator of the second-order total generalized variation,
    argmin_{x, r} 1/2 ||x - y||^2 + lambda1 ||r||_{1,2} + lambda2 ||J(Dx - r)||_{1,F}, lambda1 = 0.1 ths, lambda2 = 0.15 ths."""

    def __init__(self, verbose: bool = False, n_it_max: int = 1000, crit: float = 1e-5, x2: torch.Tensor = None,
                 u2: torch.Tensor = None, r2: torch.Tensor = None, ths: float | torch.Tensor = None, check_every: int = 16):
        super().__init__()
        self.verbose = verbose
        self.n_it_max = n_it_max
        self.crit = crit
        self.restart = True
        self.ths = ths
        self.tau = 0.01
        self.rho = 1.99
        self.x2 = x2
        self.r2 = r2
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
                                      "(3-D total generalized variation is not implemented)")
        _no_grad_guard_tv(type(self).__name__, y, ths)
        restart = self.restart or self.x2 is None or self.x2.shape != y.shape
        if restart:
            x2 = y
            r2 = torch.zeros((*y.shape, 2), device=y.device, dtype=y.dtype)
            u2 = torch.zeros((*y.shape, 4), device=y.device, dtype=y.dtype)
            self.restart = False
        else:
            x2, r2, u2 = self.x2, self.r2, self.u2
        if isinstance(ths, torch.Tensor):
            ths = ths.squeeze()
        lam = self._handle_sigma(ths, batch_size=y.size(0), ndim=y.ndim, device=y.device, dtype=y.dtype)
        # the reference's per-sample constants, formed by torch exactly as tgv.py:124-143 and :77 form them
        tl1 = self.tau * (lam * 0.1)
        l2 = lam * 0.15
        stats = {}
        with torch.no_grad():
            x2, r2, u2, self.n_iter = ops.tgv_prox(y, tl1.reshape(-1), l2.reshape(-1), x2, r2, u2, tau=self.tau, rho=self.rho,
                                                   n_it_max=self.n_it_max, crit=self.crit, check_every=self.check_every,
                                                   stats=stats)
        if stats["converged"]:
            self.has_converged = True
            if self.verbose:
                print("TGV prox reached convergence")
        elif self.verbose and self.n_it_max > 0:
            print("The algorithm did not converge, stopped after " + str(self.n_it_max) + " iterations.")
        self.x2 = x2.to(y.dtype).detach()
        self.r2 = r2.to(y.dtype).detach()
        self.u2 = u2.to(y.dtype).detach()
        return self.x2

    @staticmethod
    def nabla(x: torch.Tensor) -> torch.Tensor:
        return TVDenoiser.nabla(x)

    @staticmethod
    def nabla_adjoint(x: torch.Tensor) -> torch.Tensor:
        return TVDenoiser.nabla_adjoint(x)

    @staticmethod
    def epsilon(I: torch.Tensor) -> torch.Tensor:  # noqa: E741  (the reference's name)
        if I.ndim not in [5, 6]:
            raise ValueError(f"Input tensor must be 5D or 6D, got {I.ndim}D")
        return ops.tgv_epsilon(I)

    @staticmethod
    def epsilon_adjoint(G: torch.Tensor) -> torch.Tensor:
        if G.ndim not in [5, 6]:
            raise ValueError(f"Input tensor must be 5D or 6D, got {G.ndim}D")
        return ops.tgv_epsilon_adjoint(G)
