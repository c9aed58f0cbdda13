"""Every launch path of the direct blur kernels on the GPU against the fp64 restatement (tests/blur_ref64.py): TMA-box and
mapped-loop staging of one tile, ragged last tiles and a 256² image whose interior and border tiles stage differently; every
`shift` (w = 1 .. 8, h != w, even filters); the paths that switch TMA off for a whole call (W % 4 != 0, an input off 16-byte
alignment, box edges above 256, DINVK_NO_TMA_STAGING); cfg5 (32 x 1024², 31 x 31), 63 x 63 and the shared-memory acceptance
boundary in both directions; images smaller than the filter; per-sample / per-channel filters; the 65535-plane grid; an empty
batch; and NaN / ±Inf inside tiles, on every border and on a tile seam.  The case table and its assertions live in
tests/blur_path_cases.py; tests/test_emul_blur_paths.py runs the same table through the host emulation.

The kernel census runs every row's call under torch.profiler and checks that each row launched the kernels it names, and that
the table as a whole reaches both kernels."""
import re
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import blur_path_cases as T  # noqa: E402

pytestmark = pytest.mark.gpu

CENSUS = [T.K_CORR, T.K_FOLD]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row, dev):
    res = T.check_row(row, dev)
    print(f"\n{row.name}: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in res.items()))


def test_kernel_census(dev):
    """every row launched the kernels it names (each row's call alone under its own profile), and the table as a whole reaches
    both kernels"""
    from torch.profiler import ProfilerActivity, profile

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return {re.sub(r"\s+", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}

    probe = torch.ones(1024, device=dev)
    if not kernels(lambda: probe.mul_(2)):  # (the first profile also initialises the tracer)
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable); the numeric tests do not depend on it")
    seen = set()
    wrong = []
    for row in T.ROWS:
        if row.error or not row.kernels:
            continue
        case = T.Case(row, dev)
        with T._env(row.env):
            call = case.make_call()
            for _ in range(3):  # the tracer now and then delivers no record at all for a profile: that is no evidence, retry
                names = kernels(call)
                if names:
                    break
        seen |= names
        miss = [k for k in row.kernels if not any(k in n for n in names)]
        extra = [n for n in names if "blur" in n and not any(k in n for k in row.kernels)]
        if miss or extra:
            wrong.append((row.name, miss, extra, sorted(names)))
    missing = [k for k in CENSUS if not any(k in n for n in seen)]
    print("\n".join(["", "blur kernels launched by the table:"] + sorted(n for n in seen if "blur" in n)))
    assert not wrong, f"rows that did not launch exactly their kernels: {wrong}"
    assert not missing, f"kernels not launched by the table: {missing}"
