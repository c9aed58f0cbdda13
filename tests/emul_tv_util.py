"""helpers shared by the TV and TGV emulation tests: the emulation library of deepinv_b200/csrc/tv.cu (one per choice of
tile edge and iterations per launch) and test inputs"""
import ctypes as C
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent / "emul"))

from deepinv_b200 import _ffi  # noqa: E402

_libs = {}


def lib(tv=None, tgv=None):
    """the emulation library, built with the TV prox's and the TGV prox's (tile, iterations per launch) if given"""
    defines = {}
    if tv:
        defines.update(DINVK_TV_TILE=tv[0], DINVK_TV_BLOCK=tv[1])
    if tgv:
        defines.update(DINVK_TGV_TILE=tgv[0], DINVK_TGV_BLOCK=tgv[1])
    key = tuple(sorted(defines.items()))
    if key not in _libs:
        from build_emul_tv import build

        _libs[key] = _ffi.bind(C.CDLL(str(build(**defines))), required=False)
    return _libs[key]


def _p(t):
    return C.c_void_p(t.data_ptr())


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def image(B, Cc, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    base = torch.linspace(0, 1, W).expand(H, W) + torch.linspace(0, 0.5, H)[:, None]
    return (base + 0.3 * torch.randn(B, Cc, H, W, generator=g)).float()
