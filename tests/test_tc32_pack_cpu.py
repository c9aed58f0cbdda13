"""CPU checks of the split-operand formats and of the weight packings the fp32-grade tensor-core kernels consume
(deepinv_b200/models/tc_engine.py, csrc/conv_tc32.cu).  The kernels themselves need an H100 (tests/test_gpu_tc32.py); what can be
pinned without one is the ARITHMETIC CONTRACT they implement: every operand is hi + lo, the GEMM evaluates hi*hi + hi*lo + lo*hi, and
the K order of each packed weight matrix matches the order in which the kernel walks taps and channel blocks.  Each test restates the
kernel's contraction in torch (fp64 accumulation) from the PACKED tensors and compares it with the reference convolution the layer
replaces (deepinv/models/drunet.py:323-433: conv3x3 / strided conv2x2 / transposed conv2x2)."""
import pytest
import torch
import torch.nn.functional as F

from deepinv_b200.models.tc_engine import (_pack3x3_slab_tc32, _pack3x3_tc32, _pack_down_tc32, _pack_tc32, _pack_up_tc32, _rna_tf32)

CORR = {0: 1.0, 1: 2.0 ** -11}
CH = {0: 16, 1: 32}


def split_act(x: torch.Tensor, fmt: int):
    """(B,C,H,W) fp32 -> (hi, lo) fp64 tensors of the same shape, the values the store path of the kernels writes
    (conv_tc32.cu::store_split): tf32 hi + exact fp32 remainder, or fp16 hi + fp16 remainder scaled by 2^11"""
    if fmt == 0:
        hi = _rna_tf32(x)
        return hi.double(), (x - hi).double()
    hi = x.to(torch.float16)
    lo = ((x - hi.float()) * 2048.0).to(torch.float16)
    return hi.double(), lo.double() * CORR[1]


def unpack(wp: torch.Tensor, fmt: int):
    """packed (2*rows, K): per 64 rows [hi(64); lo(64)] -> (hi, lo) fp64 (rows, K), lo already weighted"""
    r2, K = wp.shape
    g = wp.double().view(r2 // 128, 2, 64, K)
    return g[:, 0].reshape(-1, K), g[:, 1].reshape(-1, K) * CORR[fmt]


def three_products(a_hi, a_lo, w_hi, w_lo):
    """what the two MMA streams accumulate: main = a_hi w_hi, corr = a_hi w_lo + a_lo w_hi (the lo*lo term is dropped)"""
    return a_hi @ w_hi.T + (a_hi @ w_lo.T + a_lo @ w_hi.T)


@pytest.mark.parametrize("fmt", [0, 1])
def test_split_formats_reconstruct(fmt):
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(4096, generator=gen) * torch.logspace(-6, 3, 4096)
    hi, lo = split_act(x, fmt)
    err = ((hi + lo) - x.double()).abs()
    if fmt == 0:
        assert torch.equal((hi + lo).float(), x)          # tf32 split: the remainder is exact, hi + lo == v bit for bit
    else:
        # fp16 split: 11 + 11 bits relative, with an absolute floor of 2^-35 (the scaled remainder of a value below 6e-5 is an
        # fp16 subnormal: spacing 2^-24 / 2^11)
        assert (err <= 2.0 ** -21 * x.double().abs() + 2.0 ** -35).all()
    w = torch.randn(128, 48, generator=gen)
    w_hi, w_lo = unpack(_pack_tc32(w, fmt), fmt)
    assert ((w_hi + w_lo) - w.double()).abs().max() < 2.0 ** -20 * w.abs().max()


@pytest.mark.parametrize("fmt", [0, 1])
def test_pertap_3x3_packing(fmt):
    """conv_tc32_kernel, 3x3: GEMM column k = (ky*3 + kx) * Cin + c"""
    gen = torch.Generator().manual_seed(1)
    ci, co = 64, 128
    x = torch.randn(1, ci, 6, 7, generator=gen)
    w = torch.randn(co, ci, 3, 3, generator=gen) / 24
    w_hi, w_lo = unpack(_pack3x3_tc32(w, fmt), fmt)
    x_hi, x_lo = split_act(x, fmt)
    cols = lambda t: F.unfold(t, 3, padding=1).view(1, ci, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * ci)   # rows = pixels, k = tap*Cin + c
    out = three_products(cols(x_hi), cols(x_lo), w_hi, w_lo).T.reshape(1, co, 6, 7)
    ref = F.conv2d(x.double(), w.double(), padding=1)
    assert (out - ref).norm() / ref.norm() < 5e-7


@pytest.mark.parametrize("fmt", [0, 1])
def test_slab_3x3_packing(fmt):
    """conv_tc32_slab_kernel: per channel block cb five weight tiles (tap pairs; the tenth tap slot is zero), inside a tile
    [tap even CH | tap odd CH]: column ((cb*5 + tap/2)*2 + tap%2)*CH + c%CH"""
    gen = torch.Generator().manual_seed(2)
    ci, co, ch = 64, 64, CH[fmt]
    x = torch.randn(2, ci, 5, 9, generator=gen)
    w = torch.randn(co, ci, 3, 3, generator=gen) / 24
    wp = _pack3x3_slab_tc32(w, fmt)
    assert wp.shape == (2 * co, 10 * ci)
    w_hi, w_lo = unpack(wp, fmt)
    x_hi, x_lo = split_act(x, fmt)
    nb = ci // ch

    def cols(t):   # the kernel's walk: channel block, tap pair, parity, channel
        u = F.unfold(t, 3, padding=1).view(2, nb, ch, 9, -1)                       # (B, cb, c, tap, pix)
        u = torch.cat([u, torch.zeros(2, nb, ch, 1, u.shape[-1], dtype=u.dtype)], 3)  # tap 9: the zero slot
        return u.view(2, nb, ch, 5, 2, -1).permute(0, 5, 1, 3, 4, 2).reshape(-1, nb * 10 * ch)
    out = three_products(cols(x_hi), cols(x_lo), w_hi, w_lo).view(2, 5 * 9, co).permute(0, 2, 1).reshape(2, co, 5, 9)
    ref = F.conv2d(x.double(), w.double(), padding=1)
    assert (out - ref).norm() / ref.norm() < 5e-7
    # the padding columns of the weight matrix are zero in both halves
    pad = wp.view(2 * co, nb, 5, 2, ch)[:, :, 4, 1, :]
    assert torch.count_nonzero(pad) == 0


@pytest.mark.parametrize("fmt", [0, 1])
def test_down_and_up_2x2_packing(fmt):
    """strided 2x2 (k = (dy*2 + dx)*Cin + c, rows = Cout) and transposed 2x2 (rows = (dy*2 + dx)*Cout + co, k = Cin: one GEMM
    column block per output phase, conv_tc32_kernel mode 2)"""
    gen = torch.Generator().manual_seed(3)
    ci, co = 64, 128
    x = torch.randn(1, ci, 6, 8, generator=gen)
    wd = torch.randn(co, ci, 2, 2, generator=gen) / 16
    w_hi, w_lo = unpack(_pack_down_tc32(wd, fmt), fmt)
    x_hi, x_lo = split_act(x, fmt)
    cols = lambda t: F.unfold(t, 2, stride=2).view(1, ci, 4, -1).permute(0, 3, 2, 1).reshape(-1, 4 * ci)
    out = three_products(cols(x_hi), cols(x_lo), w_hi, w_lo).T.reshape(1, co, 3, 4)
    ref = F.conv2d(x.double(), wd.double(), stride=2)
    assert (out - ref).norm() / ref.norm() < 5e-7

    wu = torch.randn(co, ci, 2, 2, generator=gen) / 12          # ConvTranspose2d weight: (Cin = co, Cout = ci, 2, 2)
    xu = torch.randn(1, co, 3, 4, generator=gen)
    u_hi, u_lo = unpack(_pack_up_tc32(wu, fmt), fmt)             # rows = (dy*2+dx)*Cout + o
    a_hi, a_lo = split_act(xu, fmt)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(-1, co)
    g = three_products(flat(a_hi), flat(a_lo), u_hi, u_lo).view(3, 4, 2, 2, ci)   # (y, x, dy, dx, o)
    out = g.permute(4, 0, 2, 1, 3).reshape(1, ci, 6, 8)
    ref = F.conv_transpose2d(xu.double(), wu.double(), stride=2)
    assert (out - ref).norm() / ref.norm() < 5e-7


def test_dropped_lo_lo_term_is_negligible_and_needed_terms_are_not():
    """error budget of the scheme on a DRUNet-sized contraction (K = 9 * 64): three products are 3e-7 from the exact result, the
    main product alone (plain fp16 operands) is 1e-4 .. 1e-3 away — the correction stream is what buys the tolerance"""
    gen = torch.Generator().manual_seed(4)
    a = torch.randn(256, 576, generator=gen).abs()      # post-ReLU activations: no cancellation, the hard case for a bias
    w = torch.randn(64, 576, generator=gen) / 24
    a_hi, a_lo = split_act(a, 1)
    w_hi, w_lo = unpack(_pack_tc32(w, 1), 1)
    exact = a.double() @ w.double().T
    three = three_products(a_hi, a_lo, w_hi, w_lo)
    main = a_hi @ w_hi.T
    assert (three - exact).norm() / exact.norm() < 5e-7
    assert (main - exact).norm() / exact.norm() > 5e-5
