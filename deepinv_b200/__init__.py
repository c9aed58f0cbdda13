"""deepinv_b200 — H100-native (sm_90a) drop-in for DeepInverse's physics-operator hot path.

Public surface mirrors `deepinv`: `deepinv_b200.physics`, `.optim`, `.models`, `.sampling`,
`.unfolded`.  All arithmetic runs in libdinvk.so (hand-written CUDA behind the C ABI in
include/dinvk.h); there is no CPU or PyTorch-operator fallback.
"""
from . import datasets, models, optim, physics, sampling, unfolded  # noqa: F401
from ._lib import DinvkError, get_lib, launch_count  # noqa: F401

__version__ = "0.1.0"
