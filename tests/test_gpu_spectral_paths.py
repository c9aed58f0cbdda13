"""Every launch path of `dinvk_spectral` on the GPU against the fp64 contract (tests/spectral_ref64.py) and, for BlurFFT, the oracle
in float64: FastMRI knee (640 x 368 / 372, single and 15 coils) and brain (640 x 320, 16 coils), 8- and 4-column strips and the
hand-off past the tile budget, row passes at 512 / 1024 threads, the 15-element budget of radix-3/5 plans, the fast kernels at
128 / 512 / 1024 and their geometric fallbacks, an odd smooth size, operands off 16-byte alignment, every gmode / c_batch / the
full epilogue per kernel family, the elementwise-only call, and BlurFFT at 1080p and 720p.  The case table and its assertions
live in tests/spectral_path_cases.py; tests/test_emul_spectral_paths.py runs the same table through the host emulation.

A kernel census runs every row once under torch.profiler and checks that the union of the launched kernels contains every
spectral kernel instantiation the table is meant to reach, so a later dispatch change cannot move a row onto an already-tested
path unnoticed."""
import re
import sys
from pathlib import Path

import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import spectral_path_cases as T  # noqa: E402

pytestmark = pytest.mark.gpu

# kernel names (demangled, spaces removed) the table must launch
CENSUS = [
    "spectral_pass_kernel<true,256>", "spectral_pass_kernel<true,512>", "spectral_pass_kernel<true,1024>",
    "spectral_pass_kernel<false,256>", "spectral_pass_kernel<false,512>", "spectral_pass_kernel<false,1024>",
    "spectral_fast_kernel<9,true,512,16>", "spectral_fast_kernel<9,false,256,8>", "spectral_fast_kernel<7,false,256,32>",
    "spectral_fast_kernel<10,true,1024,16>", "spectral_fast_kernel<10,false,256,4>",
    "dft_axis_naive_kernel", "coil_combine_kernel",
    "sp::sp_pass1", "sp::sp_pass2", "sp::sp_row_fused", "sp320::sp320_pass1", "sp320::sp320_pass2",
]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("row", T.ROWS, ids=[r.name for r in T.ROWS])
def test_path(row, dev):
    res = T.check_row(row, dev)
    print(f"\n[{row.path}] {row.name}: " + ", ".join(f"{k} {v:.3g}" for k, v in res.items()))


def test_kernel_census(dev):
    from torch.profiler import ProfilerActivity, profile

    cases = [T.Case(r, dev) for r in T.ROWS]
    # the 256² / 320² rows off alignment also run their aligned twin, which the pipelined kernels take
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in cases:
            c.run()
            if c.row.offset:
                c.run_aligned()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    if not names:
        pytest.skip("torch.profiler recorded no CUDA kernels on this machine (CUPTI unavailable); the numeric tests do not depend on it")
    flat = {re.sub(r"\s+", "", n) for n in names}
    missing = [k for k in CENSUS if not any(k in n for n in flat)]
    spectral = sorted(n for n in flat if "dinvk" in n)
    print("\n".join(["", "spectral kernels launched by the table:"] + spectral))
    assert not missing, f"kernels not launched by the table: {missing}; launched: {spectral}"
