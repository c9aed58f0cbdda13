"""Host-emulated twin of tests/test_gpu_blur3d.py's launch-path rows: the case table of tests/blur3d_path_cases.py through the
emulation build of the kernel library, with the same tolerances and launch counts.  Rows that would take more than a few seconds
on the host run at the (B, C, D, H, W) the table gives them, on the same host branch.  The emulation has no TMA (every tile stages
by the mapped loop), so the TMA-against-loop equality is checked on the GPU only."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import blur3d_path_cases as T  # noqa: E402
import radon_path_cases as RT  # noqa: E402


@pytest.fixture(autouse=True)
def emul_backend(monkeypatch):
    from deepinv_b200 import ops

    RT.install_emul(monkeypatch.setattr)
    yield
    ops._ws_cache.clear()


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row):
    if row.gpu_only:
        pytest.skip(row.gpu_only)
    T.check_row(row, torch.device("cpu"), emulated=True)


def test_table_coverage():
    """every shift 0 .. 3 in each direction on TMA-eligible rows, every layout, both stagings, every padding in both directions"""
    ok = [r for r in T.ROWS if not r.error and r.B]
    tma = [r for r in ok if T.staging(r, r.W) == "tma"]
    for tr in (False, True):
        assert {T.layout(tr, r.pad, r.h, r.w)[2] for r in tma if r.transpose == tr} == {0, 1, 2, 3}, tr
    assert {T.layout(r.transpose, r.pad, r.h, r.w)[:2] for r in ok} == {(T.ZT, 2), (T.ZT, 1), (1, 1)}
    assert any(T.staging(r, r.W) == "loop" and not r.env and r.call != "raw" for r in ok)
    assert {(r.pad, r.call) for r in ok} >= {(p, c) for p in T.PADS for c in ("A", "At")}
    assert T.layout(False, "circular", T.N_ONE, T.N_ONE) is not None and T.layout(True, "circular", T.N_ONE + 1, T.N_ONE + 1) is None
