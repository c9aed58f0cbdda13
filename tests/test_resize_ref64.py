"""The fp64 restatement of MATLAB-bicubic imresize (tests/resize_ref64.py) against the reference's golden vectors
(tests/golden/resize_*.npz, deepinv 0.4.1 on CPU), and the library's host-side tables against the restatement.  CPU only."""
import pytest
import torch

import resize_ref64 as R
from conftest import golden_names, load_golden, rel_err

DOWN = [n for n in golden_names("resize_f") if n != "resize_f15_aa"]


@pytest.mark.parametrize("name", DOWN)
def test_restatement_matches_reference(name):
    g = load_golden(name)
    f, aa = int(g["factor"]), bool(int(g["aa"]))
    assert rel_err(R.imresize(g["x"], 1 / f, aa), g["y"]) < 1e-6
    assert rel_err(R.downsample_adjoint(g["v"], f, aa), g["At"]) < 1e-6


def test_restatement_upscaling_and_sizes():
    g = load_golden("resize_up2")
    x = g["x"]
    assert rel_err(R.imresize(x, 2.0), g["up2"]) < 1e-6
    assert rel_err(R.imresize(x, 2.0, antialiasing=False), g["up2_noaa"]) < 1e-6
    for key, (ho, wo) in (("up_sizes", (25, 17)), ("down_sizes", (6, 9))):
        MH, MW = R.matrix(11, ho, ho / 11), R.matrix(14, wo, wo / 14)
        assert rel_err(R.apply(x, MH, MW), g[key]) < 1e-6


@pytest.mark.parametrize("name", golden_names("resize_tiny_"))
def test_restatement_tiny_images_raise(name):
    g = load_golden(name)
    assert int(g["err"]) == 4  # IndexError
    with pytest.raises(IndexError):
        R.imresize(g["x"], 1 / int(g["factor"]))


@pytest.mark.parametrize("n,scale,aa", [(23, 0.5, True), (17, 1 / 3, True), (37, 0.25, True), (30, 0.5, False), (11, 2.0, True),
                                        (14, 25 / 14, True), (64, 0.125, True), (9, 0.6, True)])
def test_tables_restate_the_matrix(n, scale, aa):
    """the library's per-axis tables (forward band and transposed CSR) assemble to the fp64 matrix up to fp32 weights"""
    import math

    from deepinv_b200.physics.imresize import axis_table

    m = math.ceil(n * scale)
    t = axis_table(n, m, scale, aa)
    j = t.base.long()[:, None] + torch.arange(t.k)[None, :]
    j = torch.where(j < 0, -1 - j, torch.where(j >= n, 2 * n - 1 - j, j))
    M = torch.zeros(m, n, dtype=torch.float64).scatter_add_(1, j, t.weight.double())
    ref = R.matrix(n, m, scale, aa)
    assert float((M - ref).abs().max()) < 1e-6
    # the CSR holds every (output, tap) pair once, sorted by input then output
    assert int(t.ptr[-1]) == m * t.k and t.out.numel() == m * t.k
    Mt = torch.zeros(n, m, dtype=torch.float64)
    for i in range(n):
        a, b = int(t.ptr[i]), int(t.ptr[i + 1])
        assert torch.all(t.out[a:b][1:] >= t.out[a:b][:-1])
        Mt[i].index_add_(0, t.out[a:b].long(), t.wt[a:b].double())
    assert torch.equal(Mt, M.t())
