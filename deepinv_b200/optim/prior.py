"""Priors (deepinv/optim/prior.py:13-109): PnP prox = denoiser(x, sigma)."""
from __future__ import annotations

import torch
import torch.nn as nn


class Prior(nn.Module):
    def __init__(self, g=None):
        super().__init__()
        self._g = g
        self.explicit_prior = g is not None

    def fn(self, x, *args, **kwargs):
        return self._g(x, *args, **kwargs)

    def forward(self, x, *args, **kwargs):
        return self.fn(x, *args, **kwargs)

    def grad(self, x, *args, **kwargs):
        with torch.enable_grad():
            x = x.requires_grad_()
            return torch.autograd.grad(self.fn(x, *args, **kwargs).sum(), x, create_graph=True)[0]

    def prox(self, x, *args, gamma=1.0, **kwargs):
        raise NotImplementedError

    def prox_conjugate(self, x, *args, gamma=1.0, lamb=1.0, **kwargs):
        """prox of (lamb g)^* by Moreau's identity (potential.py:120-133): x - gamma prox_{lamb/gamma g}(x / gamma)"""
        return x - gamma * self.prox(x / gamma, *args, gamma=lamb / gamma, **kwargs)


class ZeroPrior(Prior):
    def __init__(self):
        super().__init__()
        self.explicit_prior = True

    def fn(self, x, *args, **kwargs):
        return torch.zeros(x.shape[0], device=x.device)

    def grad(self, x, *args, **kwargs):
        return torch.zeros_like(x)

    def prox(self, x, *args, gamma=1.0, **kwargs):
        return x


class PnP(Prior):
    """Plug-and-play prior: prox_{gamma g}(x) = D_sigma(x)  (prior.py:86-109)"""

    def __init__(self, denoiser, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.denoiser = denoiser
        self.explicit_prior = False

    def prox(self, x, sigma_denoiser, *args, **kwargs):
        return self.denoiser(x, sigma_denoiser)


class RED(Prior):
    """Regularisation by denoising: grad g(x) = x - D_sigma(x)  (prior.py:112-135); one axpby after the denoiser"""

    def __init__(self, denoiser, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.denoiser = denoiser
        self.explicit_prior = False

    def grad(self, x, sigma_denoiser, *args, **kwargs):
        d = self.denoiser(x, sigma_denoiser)
        if torch.is_grad_enabled() and (x.requires_grad or d.requires_grad):
            return x - d
        from .. import ops

        return ops.axpbypcz(x, 1.0, d, -1.0)


class Tikhonov(Prior):
    """g(x) = 1/2 ||x||^2 (prior.py:227-266): grad = x, prox = x / (1 + gamma)"""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.explicit_prior = True

    def fn(self, x, *args, **kwargs):
        return 0.5 * (x.reshape(x.shape[0], -1) ** 2).sum(-1)

    def grad(self, x, *args, **kwargs):
        return x

    def prox(self, x, *args, gamma=1.0, **kwargs):
        return (1 / (gamma + 1)) * x


class TVPrior(Prior):
    """Total variation g(x) = ||Dx||_{1,2} (prior.py:485-572).  prox = TVDenoiser(x, ths=gamma) with crit=def_crit; fn, grad,
    nabla and nabla_adjoint are one libdinvk launch each (fn: two).  prox_conjugate comes from Prior (Moreau), so PDCP runs."""

    _l1 = False

    def __init__(self, def_crit=1e-8, n_it_max=1000, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.explicit_prior = True
        from ..models.tv import TVDenoiser, TVL1Denoiser

        self.TVModel = (TVL1Denoiser if self._l1 else TVDenoiser)(crit=def_crit, n_it_max=n_it_max)

    def fn(self, x, *args, **kwargs):
        from .. import ops

        return ops.tv_fn(x, l1=self._l1)

    def prox(self, x, *args, gamma=1.0, **kwargs):
        return self.TVModel(x, ths=gamma)

    def nabla(self, x):
        return self.TVModel.nabla(x)

    def nabla_adjoint(self, x):
        return self.TVModel.nabla_adjoint(x)

    def grad(self, x, *args, **kwargs):
        """subgradient -div(Dx / |Dx|), the zero element where Dx = 0 (prior.py:544-572)"""
        from .. import ops

        return ops.tv_grad(x)


class TVL1Prior(TVPrior):
    """g(x) = ||Dx||_1 (prior.py:575-611); prox by TVL1Denoiser, grad inherited from TVPrior as in the reference"""

    _l1 = True
