"""Host-emulated twin of tests/test_gpu_spectral_paths.py: the same case table (tests/spectral_path_cases.py) through the emulation
build of the kernel library, with the same tolerances and launch counts.  Rows that would take more than a couple of seconds on the
host run at the smaller size the table gives them, chosen to keep the row on the same launch path (same kernel family, launch count,
strip width or thread count)."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import spectral_path_cases as T  # noqa: E402


@pytest.fixture(autouse=True)
def emul_backend(monkeypatch):
    from emul_util import emul_lib

    from deepinv_b200 import ops

    lib = emul_lib()

    def check(rc):
        assert rc == 0, lib.dinvk_last_error()

    monkeypatch.setattr(ops, "_require_cuda", lambda *ts: torch.device("cpu"))
    monkeypatch.setattr(ops, "_stream", lambda dev: None)
    monkeypatch.setattr(ops, "get_lib", lambda: lib)
    monkeypatch.setattr(ops, "check", check)
    ops._ws_cache.clear()
    yield
    ops._ws_cache.clear()


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row):
    T.check_row(row, torch.device("cpu"), emulated=True)
