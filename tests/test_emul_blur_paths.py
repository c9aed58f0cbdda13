"""Host-emulated twin of tests/test_gpu_blur_paths.py: the same case table (tests/blur_path_cases.py) through the emulation build of
the kernel library, with the same tolerances and launch counts.  Rows that would take more than a few seconds on the host run at
the (B, H, W) the table gives them, on the same host branch.  The emulation has no TMA (every tile stages by the mapped loop), so
the TMA-against-loop equality is checked on the GPU only; the 65535-plane success rows are GPU-only."""
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import blur_path_cases as T  # noqa: E402
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
    """the table reaches every shift 0 .. 3 in each direction on TMA-eligible rows, both stagings, and a boundary derived from the
    budget formula that A and A^T share for every padding"""
    tma = [r for r in T.ROWS if not r.error and r.B and T.staging(r, r.B, r.H, r.W) == "tma"]
    for tr in (False, True):
        shifts = {T.layout(r.transpose, r.pad, r.h, r.w)[0] for r in tma if r.transpose == tr}
        assert shifts == {0, 1, 2, 3}, (tr, shifts)
    assert any(r.pad in T.SAME[:3] for r in tma)  # tiles that take the box inside and the loop at the border
    assert any(T.staging(r, r.B, r.H, r.W) == "loop" and not r.env and r.call != "raw" for r in T.ROWS if not r.error)
    for shape, n in (((lambda n: (n, n)), T.N_SQ), ((lambda n: (1, n)), T.N_ROW), ((lambda n: (n, 1)), T.N_COL)):
        for pad in T.BR.PADS:
            for tr in (False, True):
                assert T.layout(tr, pad, *shape(n)) is not None and T.layout(tr, pad, *shape(n + 1)) is None
    accepted = {(r.h, r.w) for r in T.ROWS if r.name.startswith("accept")}
    rejected = {(r.h, r.w) for r in T.ROWS if r.name.startswith("reject")}
    assert {(T.N_SQ, T.N_SQ), (1, T.N_ROW), (T.N_COL, 1)} <= accepted
    assert rejected == {(T.N_SQ + 1, T.N_SQ + 1), (1, T.N_ROW + 1), (T.N_COL + 1, 1)}
