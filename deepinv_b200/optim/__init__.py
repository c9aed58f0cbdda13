from .data_fidelity import L2, DataFidelity, ZeroFidelity  # noqa: F401
from .dpir import DPIR, get_DPIR_params  # noqa: F401
from .graphed import GraphedIteration, GraphedSolve, HostStreamedIteration  # noqa: F401
from .linear import bicgstab, conjugate_gradient, least_squares, lsqr, minres  # noqa: F401
from .optim_iterators import (ADMMIteration, CPIteration, DRSIteration, FISTAIteration, GDIteration, HQSIteration,  # noqa: F401
                              OptimIterator, PGDIteration)
from .optimizers import (ADMM, DRS, FISTA, GD, HQS, PDCP, PGD, AndersonAccelerationConfig, BacktrackingConfig, BaseOptim,
                         DEQConfig,  # noqa: F401
                         create_iterator,
                         optim_builder)
from .prior import RED, PnP, Prior, Tikhonov, TVL1Prior, TVPrior, ZeroPrior  # noqa: F401
