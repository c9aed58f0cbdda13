"""Host-emulated twin of tests/test_gpu_radon_paths.py: the same case table (tests/radon_path_cases.py) through the emulation
build of the kernel library, with the same tolerances and launch counts.  Rows that would take more than a few seconds on the
host run at the (W, A) the table gives them, chosen to keep the row on the same launch path.  The emulation has no TMA (the
"TMA" forward rows stage by the mapped loop here too) and no 48 KB shared-memory limit, so the rows that exist to cross that
limit are GPU-only."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import radon_path_cases as T  # noqa: E402


@pytest.fixture(autouse=True)
def emul_backend(monkeypatch):
    from deepinv_b200 import ops

    T.install_emul(monkeypatch.setattr)
    yield
    ops._ws_cache.clear()


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row):
    if row.gpu_only:
        pytest.skip(row.gpu_only)
    T.check_row(row, torch.device("cpu"), emulated=True)


def test_ramp_fft_form():
    """DINVK_RAMP_FFT: mean subtraction, row pass, box response, odd row counts, with and without a workspace (child process)"""
    rep = T.run_fft_rows(emulated=True)
    print(rep)
    T.check_fft_report(rep)
