"""Loader of libdinvk.so — the only compute backend of this package.

There is deliberately no fallback: if the shared object is missing or CUDA is unavailable, every
operator raises.  (The CPU emulation under tests/emul is test infrastructure and is never loaded
from here.)
"""
from __future__ import annotations

import ctypes
import threading
from pathlib import Path

from . import _ffi

_LIB_PATH = Path(__file__).resolve().parent / "libdinvk.so"
_lock = threading.Lock()
_lib = None


class DinvkError(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def get_lib() -> ctypes.CDLL:
    """Return the bound library, loading it on first use."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not _LIB_PATH.exists():
                    raise DinvkError(
                        f"{_LIB_PATH} is missing: build it with `python -m deepinv_b200.build` "
                        "(deepinv_b200 has no CPU or PyTorch fallback)."
                    )
                lib = ctypes.CDLL(str(_LIB_PATH))
                _ffi.bind(lib, required=True)  # every symbol of include/dinvk.h must be exported
                if lib.dinvk_version() < 100:
                    raise DinvkError("libdinvk.so is older than this package")
                _lib = lib
    return _lib


def check(rc: int, lib: ctypes.CDLL | None = None) -> None:
    """raise the error of the library call that returned rc (of `lib`, the package's library by default)"""
    if rc != 0:
        msg = (lib or get_lib()).dinvk_last_error()
        raise DinvkError(f"libdinvk error {rc}: {msg.decode(errors='replace') if msg else ''}")


def launch_count() -> int:
    return int(get_lib().dinvk_launch_count())
