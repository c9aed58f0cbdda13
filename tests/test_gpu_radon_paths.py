"""Every launch path of the Radon family and the ramp filter on the GPU against the fp64 restatement (tests/radon_ref64.py): the
tiled kernels with TMA and mapped-loop staging (one tile, a 4-pixel last tile, cfg3 512² / 180 angles, P = 1449, circles,
C = 3, A = 1 and the 2048-angle limit), the per-ray kernels (W < 64, W % 4 == 2, odd-width circle, 2049 .. 4096 angles on
both sides of the 48 KB shared-memory line, an input off 16-byte alignment, DINVK_NO_TILED_RADON), user-given and near-axis
angles, IRadon A_adjoint and FBP, fan beam, the exact ramp kernel up to N = 8192 and its FFT form, the fixed-point range of
the tiled transpose, and NaN / ±Inf in each forward's and each transpose's input.  The case table and its assertions live in
tests/radon_path_cases.py; tests/test_emul_radon_paths.py runs the same table through the host emulation.

The kernel census runs every row's call under torch.profiler and checks that each row launched the kernel it names, and that
the table as a whole reaches every kernel of the family."""
import re
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import radon_path_cases as T  # noqa: E402

pytestmark = pytest.mark.gpu

CENSUS = [T.K_TILED_F, T.K_TILED_A, T.K_RAY_F, T.K_RAY_A, T.K_IRADON, T.K_FAN_F, T.K_FAN_A, T.K_RAMP]
CENSUS_FFT = ["ramp_mean_sub_kernel", "ramp_add_box_kernel", "spectral_pass_kernel<false"]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row, dev):
    res = T.check_row(row, dev)
    print(f"\n{row.name}: " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in res.items()))


def test_ramp_fft_form(dev):
    """DINVK_RAMP_FFT: mean subtraction, row pass, box response, odd row counts, with and without a workspace (child process),
    and the clean error past the exact kernel's N = 8192"""
    rep = T.run_fft_rows(emulated=False)
    for r in rep["rows"]:
        print(r)
    print("N = 8193:", rep["n8193"])
    T.check_fft_report(rep)
    flat = {re.sub(r"\s+", "", n) for n in rep["kernels"]}
    if not flat:
        pytest.skip("the numeric checks passed, but torch.profiler recorded no CUDA kernels in the child (CUPTI unavailable): "
                    "the FFT form's kernels are not verified")
    missing = [k for k in CENSUS_FFT if not any(k in n for n in flat)]
    assert not missing, f"FFT form: kernels not launched: {missing}; launched: {sorted(flat)}"


def test_kernel_census(dev):
    """every row launched the kernel it names, and the table as a whole reaches every kernel of the family (each row's call alone
    under its own profile: one profile around a whole check_row missed the kernels of some rows)"""
    from torch.profiler import ProfilerActivity, profile

    seen = set()
    wrong = []
    for row in T.ROWS:
        if row.error:
            continue
        case = T.Case(row, dev)
        with T._env(row.env):
            call = case.make_call()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call()
                torch.cuda.synchronize()
        names = {re.sub(r"\s+", "", e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if not names:
            pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable); the numeric tests do not depend on it")
        seen |= names
        want = row.kernels[:1] if row.call == "raw_A" else row.kernels  # the offset row's aligned twin is not part of its call
        miss = [k for k in want if not any(k in n for n in names)]
        if miss:
            wrong.append((row.name, miss, sorted(n for n in names if "dinvk" in n)))
    missing = [k for k in CENSUS if not any(k in n for n in seen)]
    print("\n".join(["", "Radon-family kernels launched by the table:"] + sorted(n for n in seen if "dinvk" in n)))
    assert not wrong, f"rows that did not launch their kernel: {wrong}"
    assert not missing, f"kernels not launched by the table: {missing}"
