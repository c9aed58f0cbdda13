"""GPU tests of the fp32-grade tensor-core denoiser path (precision="tc32": 3 x TF32 split operands on wgmma,
csrc/conv_tc32.cu) against fp64 / fp32 ATen convolutions and the oracle.

Tolerance: the north star's 1e-5 relative L2 for whole networks and PnP loops (the reference computes these in fp32:
deepinv/models/drunet.py:200-263, dncnn.py:121-140); single layers are held to 2e-6 against an fp64 evaluation, and the
kernel's error against fp64 must not exceed a small multiple of the error of ATen's own fp32 convolution against fp64
(the fp64-yardstick: "as close to the exact result as the reference itself")."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _to_split(x, dev, fmt=0):
    from deepinv_b200 import ops

    return ops.nchw_to_split16(x.to(dev), fmt)


def _from_split(t):
    from deepinv_b200 import ops

    return ops.split16_to_nchw(t).cpu()


def test_split16_roundtrip_is_exact(dev):
    x = torch.randn(2, 48, 9, 13) * torch.logspace(-6, 3, 48).view(1, 48, 1, 1)
    t = _to_split(x, dev)
    assert t.shape == (2, 9, 13, 3, 2, 16)
    assert torch.equal(_from_split(t), x)  # hi + lo == v exactly
    hi = t[..., 0, :].cpu()
    assert torch.equal(hi.view(torch.int32) & 0x1FFF, torch.zeros_like(hi, dtype=torch.int32))  # hi is a tf32 value
    assert (t[..., 1, :].abs().cpu() <= hi.abs() * 2.0 ** -11 + 1e-45).all()


@pytest.mark.parametrize("shape", [(2, 64, 64, 32, 48), (1, 64, 128, 16, 16), (2, 128, 128, 24, 40), (1, 256, 256, 8, 16),
                                   (1, 512, 512, 8, 16), (3, 128, 64, 9, 21), (1, 32, 64, 17, 33)])
@pytest.mark.parametrize("window", [0, 1, 3, 1000])
@pytest.mark.parametrize("fmt", [0, 1])
def test_conv3x3_tc32(shape, window, fmt, dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3_tc32

    B, Cin, Cout, H, W = shape
    if fmt == 1 and Cin % 64:
        pytest.skip("fp16 format: two 32-channel blocks per pipeline stage")
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(B, Cin, H, W, generator=gen).abs()          # post-ReLU-like: all-positive activations
    w = torch.randn(Cout, Cin, 3, 3, generator=gen) / (3 * Cin ** 0.5)
    r1, r2 = torch.randn(B, Cout, H, W, generator=gen), torch.randn(B, Cout, H, W, generator=gen)
    bias = torch.randn(Cout, generator=gen)
    wp = _pack3x3_tc32(w.to(dev), fmt)
    xs = _to_split(x, dev, fmt)
    ref64 = F.conv2d(x.double(), w.double(), padding=1)
    ref32 = F.conv2d(x, w, padding=1)
    out = _from_split(ops.conv_tc32(xs, wp, Cout, window=window))
    e_k, e_ref = rel_err(out.double(), ref64), rel_err(ref32.double(), ref64)
    assert e_k < (2e-6 if window != 1000 else 2e-5), (e_k, e_ref)
    if window != 1000:  # (1000 = never drained inside a tile: the tensor core's truncating accumulator shows, ~1e-6)
        assert e_k < max(4 * e_ref, 5e-7), (e_k, e_ref)
    out = _from_split(ops.conv_tc32(xs, wp, Cout, bias=bias.to(dev), res=_to_split(r1, dev, fmt), res2=_to_split(r2, dev, fmt), relu=True,
                                    window=window))
    ref = F.relu(F.conv2d(x.double(), w.double(), bias.double(), padding=1)) + r1.double() + r2.double()
    assert rel_err(out.double(), ref) < (2e-6 if window != 1000 else 2e-5)


@pytest.mark.parametrize("shape", [(2, 64, 64, 32, 48), (1, 64, 128, 16, 16), (2, 128, 128, 24, 40), (1, 256, 256, 8, 16),
                                   (1, 512, 512, 8, 16), (3, 128, 64, 9, 21), (1, 16, 64, 17, 33), (5, 64, 64, 40, 72)])
@pytest.mark.parametrize("window", [0, 1, 2])
@pytest.mark.parametrize("fmt", [0, 1])
def test_conv3x3_tc32_slab(shape, window, fmt, dev):
    """the halo-reuse kernel (16x16-pixel tiles, two accumulators per CTA, nine taps out of one slab)"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3_slab_tc32

    B, Cin, Cout, H, W = shape
    if fmt == 1 and Cin % 32:
        pytest.skip("fp16 format: 32-channel blocks")
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(B, Cin, H, W, generator=gen).abs()
    w = torch.randn(Cout, Cin, 3, 3, generator=gen) / (3 * Cin ** 0.5)
    r1, r2 = torch.randn(B, Cout, H, W, generator=gen), torch.randn(B, Cout, H, W, generator=gen)
    bias = torch.randn(Cout, generator=gen)
    wp = _pack3x3_slab_tc32(w.to(dev), fmt)
    xs = _to_split(x, dev, fmt)
    ref64 = F.conv2d(x.double(), w.double(), padding=1)
    ref32 = F.conv2d(x, w, padding=1)
    out = _from_split(ops.conv_tc32_slab(xs, wp, Cout, window=window))
    e_k, e_ref = rel_err(out.double(), ref64), rel_err(ref32.double(), ref64)
    assert e_k < 2e-6, (e_k, e_ref)
    if not (window == 2 and fmt == 1):  # (two fp16 blocks = k 576 per window: the truncating accumulator shows, ~1e-6)
        assert e_k < max(4 * e_ref, 5e-7), (e_k, e_ref)
    out = _from_split(ops.conv_tc32_slab(xs, wp, Cout, bias=bias.to(dev), res=_to_split(r1, dev, fmt), res2=_to_split(r2, dev, fmt), relu=True,
                                         window=window))
    ref = F.relu(F.conv2d(x.double(), w.double(), bias.double(), padding=1)) + r1.double() + r2.double()
    assert rel_err(out.double(), ref) < 2e-6


def test_conv3x3_tc32_positive_sums_no_bias(dev):
    """all-positive weights and activations: a truncating accumulator would shrink every output (negative mean error)"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3_slab_tc32, _pack3x3_tc32

    gen = torch.Generator().manual_seed(3)
    x = torch.rand(1, 512, 16, 16, generator=gen) + 0.5
    w = (torch.rand(64, 512, 3, 3, generator=gen) + 0.5) / 4608
    ref64 = F.conv2d(x.double(), w.double(), padding=1)
    # (a truncating accumulator biases the result negatively; the bias grows with the MMAs per accumulation window)
    for fn, pack, kw, lim in ((ops.conv_tc32, _pack3x3_tc32, dict(window=2), 4e-7),            # k = 64 per window
                              (ops.conv_tc32_slab, _pack3x3_slab_tc32, dict(), 1e-6),          # default: k = 144
                              (ops.conv_tc32_slab, _pack3x3_slab_tc32, dict(window=2), 2.5e-6)):  # k = 288
        out = _from_split(fn(_to_split(x, dev), pack(w.to(dev)), 64, **kw)).double()
        signed = ((out - ref64) / ref64).mean().item()
        assert abs(signed) < lim, (kw, signed)
        assert rel_err(out, ref64) < 1.2 * lim + 2e-7


@pytest.mark.parametrize("shape", [(2, 64, 128, 32, 48), (1, 128, 256, 16, 32), (1, 256, 512, 16, 16), (2, 64, 64, 10, 18)])
@pytest.mark.parametrize("fmt", [0, 1])
def test_conv2x2_tc32(shape, fmt, dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack_down_tc32, _pack_up_tc32

    B, Cin, Cout, H, W = shape
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(B, Cin, H, W, generator=gen)
    wd = torch.randn(Cout, Cin, 2, 2, generator=gen) / (2 * Cin ** 0.5)
    out = _from_split(ops.conv_tc32(_to_split(x, dev, fmt), _pack_down_tc32(wd.to(dev), fmt), Cout, kind=1))
    assert rel_err(out.double(), F.conv2d(x.double(), wd.double(), stride=2)) < 2e-6
    wt = torch.randn(Cout, Cin, 2, 2, generator=gen) / (Cout ** 0.5)  # ConvTranspose2d(Cout -> Cin) weight is (Cout, Cin, 2, 2)
    xx = torch.randn(B, Cout, H, W, generator=gen)
    out = _from_split(ops.conv_tc32(_to_split(xx, dev, fmt), _pack_up_tc32(wt.to(dev), fmt), Cin, kind=2))
    assert rel_err(out.double(), F.conv_transpose2d(xx.double(), wt.double(), stride=2)) < 2e-6


@pytest.mark.parametrize("fmt", [0, 1])
def test_head_and_tail_tc32(fmt, dev):
    from deepinv_b200 import ops

    gen = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 24, 40, generator=gen)
    wh = torch.randn(64, 3, 3, 3, generator=gen) / 5
    bh = torch.randn(64, generator=gen)
    out = _from_split(ops.conv_tc32_head(x.to(dev), wh.to(dev), bias=bh.to(dev), relu=True, fmt=fmt))
    assert rel_err(out.double(), F.relu(F.conv2d(x.double(), wh.double(), bh.double(), padding=1))) < 1e-6
    # constant fill channel (DRUNet's noise map), per-sample
    wh4 = torch.randn(64, 4, 3, 3, generator=gen) / 6
    sig = torch.tensor([0.05, 0.2])
    out = _from_split(ops.conv_tc32_head(x.to(dev), wh4.to(dev), fill=sig.to(dev), fmt=fmt))
    x4 = torch.cat([x, sig.view(2, 1, 1, 1).expand(2, 1, 24, 40)], 1)
    assert rel_err(out.double(), F.conv2d(x4.double(), wh4.double(), padding=1)) < 1e-6
    # several row segments per image (W > 32), a partial one
    x = torch.randn(1, 2, 9, 70, generator=gen)
    wh2 = torch.randn(64, 2, 3, 3, generator=gen) / 4
    out = _from_split(ops.conv_tc32_head(x.to(dev), wh2.to(dev), fmt=fmt))
    assert rel_err(out.double(), F.conv2d(x.double(), wh2.double(), padding=1)) < 1e-6
    # tail: strips of 16 / 8 / 4 columns, row chunks of 32 (one chunk, and three with a partial last one)
    for Ht, Wt in ((19, 37), (70, 45)):
        t = torch.randn(2, 64, Ht, Wt, generator=gen)
        for cout in (1, 2, 3, 4):
            wt = torch.randn(cout, 64, 3, 3, generator=gen) / 24
            bt = torch.randn(cout, generator=gen)
            add = torch.randn(2, cout, Ht, Wt, generator=gen)
            out = ops.conv_tc32_tail(_to_split(t, dev, fmt), wt.to(dev), bias=bt.to(dev), add=add.to(dev)).cpu()
            assert rel_err(out.double(), F.conv2d(t.double(), wt.double(), bt.double(), padding=1) + add.double()) < 1e-6


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_drunet_tc32_vs_oracle(precision, dev):
    """whole network, the reference configuration nc=(64,128,256,512), nb=4 (drunet.py:23-263): tc32 against the oracle
    (fp32 ATen on the CPU) at the north-star tolerance, and both against an fp64 evaluation of the same weights"""
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, pretrained=None, precision=precision).eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 2, 64, 96)
    with torch.no_grad():
        ref = R.drunet_forward(x, 0.05, sd)
        ref64 = R.drunet_forward(x.double(), 0.05, {k: v.double() for k, v in sd.items()})
        out = m.to(dev)(x.to(dev), 0.05).cpu()
        m.precision = "fp32"
        out32 = m(x.to(dev), 0.05).cpu()
    e_tc, e_simt, e_ref = rel_err(out.double(), ref64), rel_err(out32.double(), ref64), rel_err(ref.double(), ref64)
    print(f"DRUNet vs fp64: {precision} {e_tc:.2e}, fp32 CUDA-core path {e_simt:.2e}, oracle (ATen CPU fp32) {e_ref:.2e}; "
          f"tc32 vs oracle {rel_err(out, ref):.2e}")
    assert rel_err(out, ref) < 1e-5
    assert e_tc < 1e-5
    assert e_simt < 1e-5  # the fp32 CUDA-core path (the one training differentiates) at the full width


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_dncnn_tc32_vs_oracle(precision, dev):
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DnCNN(in_channels=1, out_channels=1, depth=20, nf=64, pretrained=None, precision=precision).eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 1, 40, 56)
    with torch.no_grad():
        ref = R.dncnn_forward(x, sd, depth=20)
        out = m.to(dev)(x.to(dev), 0.1).cpu()
    assert rel_err(out, ref) < 1e-5


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_pnp_pgd_tc32_vs_oracle(precision, dev):
    """the benchmark's loop (PnP-PGD, MRI, full-size DRUNet) with the tc32 denoiser, 4 iterations, against the oracle"""
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP
    from oracle import ref_ops as R

    torch.manual_seed(0)
    B, H, W = 2, 64, 64
    x = torch.randn(B, 2, H, W)
    cols = (torch.rand(B, 1, 1, W) > 0.7).float()
    cols[..., W // 2 - 3: W // 2 + 3] = 1
    mask = cols.expand(B, 2, H, W).contiguous()
    den = dinv.models.DRUNet(in_channels=2, out_channels=2, pretrained=None, precision=precision).eval()
    sd = {k: v.detach().clone() for k, v in den.state_dict().items()}
    y = R.mri_A(x, mask)
    with torch.no_grad():
        ref = R.pgd(y, lambda v: R.mri_A(v, mask), lambda v: R.mri_At(v, mask), lambda v, s: R.drunet_forward(v, s, sd), 1.0, 0.05, 4)
        physics = dinv.physics.MRI(mask=mask.to(dev), img_size=(2, H, W), device=dev)
        algo = PGD(data_fidelity=L2(), prior=PnP(den.to(dev)), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)
        out = algo(y.to(dev), physics).cpu()
    assert rel_err(out, ref) < 1e-5


def test_split32h_roundtrip_and_range(dev):
    """fp16 split: hi + lo 2^-11 reproduces v to 2^-22 relative inside the fp16 range (down to the subnormals: absolute 3e-11)"""
    from deepinv_b200 import ops

    x = torch.randn(2, 64, 9, 13) * torch.logspace(-6, 4, 64).view(1, 64, 1, 1)
    t = _to_split(x, dev, 1)
    assert t.dtype == torch.float16 and t.shape == (2, 9, 13, 2, 2, 32)
    back = _from_split(t)
    assert ((back - x).abs() <= x.abs() * 2.0 ** -21 + 1e-10).all()


def test_tc32h_overflow_is_loud(dev):
    """an activation beyond the fp16 range raises the call's overflow flag and the network answers NaN — never a silently wrong image"""
    import deepinv_b200 as dinv
    from deepinv_b200.models.tc_engine import tc_overflow

    torch.manual_seed(0)
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, pretrained=None, precision="tc32h").to(dev).eval()
    x = torch.randn(1, 2, 64, 64, device=dev)
    with torch.no_grad():
        ok = m(x, 0.05)
        assert torch.isfinite(ok).all() and not tc_overflow(m)
        bad = m(x * 3e6, 0.05)
        assert torch.isnan(bad).all() and tc_overflow(m)
        again = m(x, 0.05)       # the flag is per call: the next in-range input is served normally
        assert torch.equal(again, ok) and not tc_overflow(m)
        m.precision = "tc32"     # the tf32 format has the full fp32 range
        assert torch.isfinite(m(x * 3e6, 0.05)).all()
