from .base import Denoiser  # noqa: F401
from .dncnn import DnCNN  # noqa: F401
from .drunet import DRUNet  # noqa: F401
from .tgv import TGVDenoiser  # noqa: F401
from .tv import TVDenoiser, TVL1Denoiser  # noqa: F401
