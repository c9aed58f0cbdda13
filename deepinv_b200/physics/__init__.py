from . import functional, generator  # noqa: F401
from .blur import (Blur, BlurFFT, Downsampling, DownsamplingMatlab, SpaceVaryingBlur, TiledSpaceVaryingBlur,  # noqa: F401
                   Upsampling)
from .forward import DecomposablePhysics, LinearPhysics, Physics  # noqa: F401
from .mri import MRI, DynamicMRI, MRIMixin, MultiCoilMRI, SequentialMRI, TimeMixin  # noqa: F401
from .noise import GaussianNoise, NoiseModel, ZeroNoise  # noqa: F401
from .tomography import Tomography  # noqa: F401
from .combine import (ComposedLinearPhysics, ComposedPhysics, StackedLinearPhysics, StackedPhysics, TensorList,  # noqa: F401
                      compose, stack)
from .inpainting import Denoising, Inpainting  # noqa: F401
