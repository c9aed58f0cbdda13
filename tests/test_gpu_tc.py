"""GPU tests of the bf16 tensor-core (wgmma + TMA) denoiser path against the oracle's fp32 ATen convolutions.
Tolerance: bf16 operands with fp32 accumulation give ~2^-9 relative error per product; a single layer must agree to
5e-3 relative L2 with the fp32 result computed from the SAME bf16-rounded operands to 2e-3, and a whole
network to 3e-2 (stated per test)."""
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


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def _ref_conv(xb, wb, bias=None):
    """fp32 conv of the bf16-rounded operands (isolates kernel errors from the input rounding)"""
    return F.conv2d(xb.float(), wb.float(), bias, padding=1)


@pytest.mark.parametrize("shape", [(2, 64, 64, 32, 48), (1, 64, 128, 16, 16), (2, 128, 128, 24, 40), (1, 256, 256, 8, 16),
                                   (1, 512, 512, 8, 16), (3, 128, 64, 9, 21)])
def test_conv3x3_bf16(shape, dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3

    B, Cin, Cout, H, W = shape
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(B, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, 3, 3, generator=gen) / (3 * Cin ** 0.5)
    r1, r2 = torch.randn(B, Cout, H, W, generator=gen), torch.randn(B, Cout, H, W, generator=gen)
    xb, wb = x.to(torch.bfloat16), w.to(torch.bfloat16)
    r1b, r2b = r1.to(torch.bfloat16), r2.to(torch.bfloat16)
    w2d = _pack3x3(w.to(dev))
    # plain
    out = ops.conv3x3_bf16(_nhwc(xb).to(dev), w2d)
    ref = _ref_conv(xb, wb)
    assert rel_err(out.float().permute(0, 3, 1, 2), ref) < 4e-3  # output rounding to bf16: 2^-9
    # relu + two residuals + bias
    bias = torch.randn(Cout, generator=gen)
    out = ops.conv3x3_bf16(_nhwc(xb).to(dev), w2d, bias=bias.to(dev), res=_nhwc(r1b).to(dev), res2=_nhwc(r2b).to(dev), relu=True)
    ref = F.relu(_ref_conv(xb, wb, bias)) + r1b.float() + r2b.float()
    assert rel_err(out.float().permute(0, 3, 1, 2), ref) < 4e-3


def test_conv3x3_tail_and_layout(dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3

    gen = torch.Generator().manual_seed(1)
    x = torch.randn(2, 3, 24, 40, generator=gen)
    a = ops.nchw_to_nhwc_bf16(x.to(dev), 64, fill=0.25)
    assert a.shape == (2, 24, 40, 64)
    assert rel_err(a[..., :3].float().permute(0, 3, 1, 2), x.to(torch.bfloat16).float()) < 1e-6
    assert torch.all(a[..., 3] == 0.25) and torch.all(a[..., 4:] == 0)
    sig = torch.tensor([0.1, 0.7])
    a2 = ops.nchw_to_nhwc_bf16(x.to(dev), 64, fill=sig.to(dev))
    assert torch.allclose(a2[..., 3].float().cpu(), sig.to(torch.bfloat16).float().view(2, 1, 1).expand(2, 24, 40))
    t = torch.randn(2, 64, 24, 40, generator=gen)
    w = torch.randn(2, 64, 3, 3, generator=gen) / 24
    add, bias = torch.randn(2, 2, 24, 40, generator=gen), torch.randn(2, generator=gen)
    tb, wb = t.to(torch.bfloat16), w.to(torch.bfloat16)
    out = ops.conv3x3_bf16_tail(_nhwc(tb).to(dev), _pack3x3(w.to(dev), rows_pad=16), 2, bias=bias.to(dev), add=add.to(dev))
    assert rel_err(out, _ref_conv(tb, wb, bias) + add) < 1e-4  # fp32 output: only accumulation-order error
    back = ops.nhwc_bf16_to_nchw(_nhwc(tb).to(dev), 64)
    assert rel_err(back, tb.float()) < 1e-6


@pytest.mark.parametrize("C,fill", [(2, "batch"), (3, "scalar"), (1, None), (3, None), (4, None)])
@pytest.mark.parametrize("hw", [(24, 40), (37, 61), (128, 128)])
def test_conv3x3_head(C, fill, hw, dev):
    """dedicated head kernel (im2col rows built in shared memory, one K=64 MMA block per tile) against the fp32
    convolution of the bf16-rounded operands; covers ragged tiles (H % 4, W % 32 != 0) and the constant channel"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack_head

    H, W = hw
    B = 3
    gen = torch.Generator().manual_seed(C * 100 + H)
    x = torch.randn(B, C, H, W, generator=gen)
    ct = C + (fill is not None)
    w = torch.randn(64, ct, 3, 3, generator=gen) / (3 * ct ** 0.5)
    bias = torch.randn(64, generator=gen)
    if fill == "batch":
        fv = torch.tensor([0.1, 0.45, 0.8])
        xin = torch.cat([x, fv.view(B, 1, 1, 1).expand(B, 1, H, W)], 1)
        kw = dict(fill=fv.to(dev))
    elif fill == "scalar":
        xin = torch.cat([x, torch.full((B, 1, H, W), 0.3)], 1)
        kw = dict(fill=0.3)
    else:
        xin, kw = x, {}
    w64 = _pack_head(w.to(dev))
    assert w64 is not None and w64.shape == (64, 64)
    ref = _ref_conv(xin.to(torch.bfloat16), w.to(torch.bfloat16))
    out = ops.conv3x3_head_bf16(x.to(dev), w64, **kw)
    assert out.shape == (B, H, W, 64) and out.dtype == torch.bfloat16
    assert rel_err(out.float().permute(0, 3, 1, 2), ref) < 4e-3
    out = ops.conv3x3_head_bf16(x.to(dev), w64, bias=bias.to(dev), relu=True, **kw)
    assert rel_err(out.float().permute(0, 3, 1, 2), F.relu(ref + bias.view(1, -1, 1, 1))) < 4e-3


@pytest.mark.parametrize("cout,hw", [(1, (16, 8)), (3, (37, 61)), (2, (128, 96))])
def test_conv3x3_tail_halo(cout, hw, dev):
    """64 -> Cout <= 16 tail through the slab/halo kernel (N = 16 tile), ragged sizes"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3

    H, W = hw
    gen = torch.Generator().manual_seed(cout)
    t = torch.randn(2, 64, H, W, generator=gen)
    w = torch.randn(cout, 64, 3, 3, generator=gen) / 24
    add = torch.randn(2, cout, H, W, generator=gen)
    tb, wb = t.to(torch.bfloat16), w.to(torch.bfloat16)
    out = ops.conv3x3_bf16_tail(_nhwc(tb).to(dev), _pack3x3(w.to(dev), rows_pad=16), cout, add=add.to(dev))
    assert rel_err(out, _ref_conv(tb, wb) + add) < 1e-4
    out = ops.conv3x3_bf16_tail(_nhwc(tb).to(dev), _pack3x3(w.to(dev), rows_pad=16), cout)
    assert rel_err(out, _ref_conv(tb, wb)) < 1e-4


def test_conv2x2_bf16(dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack_down, _pack_up

    gen = torch.Generator().manual_seed(2)
    x = torch.randn(2, 64, 16, 24, generator=gen).to(torch.bfloat16)
    xa = torch.randn(2, 64, 16, 24, generator=gen).to(torch.bfloat16)
    w = (torch.randn(128, 64, 2, 2, generator=gen) / 16).to(torch.bfloat16)
    out = ops.conv2x2_bf16(_nhwc(x).to(dev), _pack_down(w.to(dev)), 128, up=False)
    assert rel_err(out.float().permute(0, 3, 1, 2), F.conv2d(x.float(), w.float(), stride=2)) < 4e-3
    wt = (torch.randn(64, 32, 2, 2, generator=gen) / 8).to(torch.bfloat16)
    out = ops.conv2x2_bf16(_nhwc(x).to(dev), _pack_up(wt.to(dev)), 32, up=True, xadd=_nhwc(xa).to(dev))  # CUDA-core variant
    assert rel_err(out.float().permute(0, 3, 1, 2), F.conv_transpose2d(x.float() + xa.float(), wt.float(), stride=2)) < 4e-3
    # tensor-core variants (channel counts multiples of 64, no fused input add)
    for (B, Cin, Cout, H, W) in [(2, 64, 128, 16, 32), (1, 128, 256, 32, 16), (2, 256, 512, 8, 16), (1, 64, 64, 18, 34)]:
        x = torch.randn(B, Cin, H, W, generator=gen).to(torch.bfloat16)
        w = (torch.randn(Cout, Cin, 2, 2, generator=gen) / (2 * Cin ** 0.5)).to(torch.bfloat16)
        out = ops.conv2x2_bf16(_nhwc(x).to(dev), _pack_down(w.to(dev)), Cout, up=False)
        assert rel_err(out.float().permute(0, 3, 1, 2), F.conv2d(x.float(), w.float(), stride=2)) < 4e-3
        wt = (torch.randn(Cout, Cin, 2, 2, generator=gen) / (Cout ** 0.5)).to(torch.bfloat16)  # (in=Cout, out=Cin)
        xx = torch.randn(B, Cout, H, W, generator=gen).to(torch.bfloat16)
        out = ops.conv2x2_bf16(_nhwc(xx).to(dev), _pack_up(wt.to(dev)), Cin, up=True)
        assert rel_err(out.float().permute(0, 3, 1, 2), F.conv_transpose2d(xx.float(), wt.float(), stride=2)) < 4e-3


def test_drunet_bf16_vs_fp32(dev):
    """whole network: bf16 tensor-core path against the oracle (fp32) with identical weights"""
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, nc=(64, 128, 128, 256), nb=2, pretrained=None, precision="bf16").eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 2, 128, 64)
    with torch.no_grad():
        ref = R.drunet_forward(x, 0.05, sd, nb=2)
        out = m.to(dev)(x.to(dev), 0.05)
        m.precision = "fp32"
        out32 = m(x.to(dev), 0.05)
    assert rel_err(out32, ref) < 1e-5
    assert rel_err(out, ref) < 3e-2


def test_dncnn_bf16_vs_fp32(dev):
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DnCNN(in_channels=1, out_channels=1, depth=6, nf=64, pretrained=None, precision="bf16").eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 1, 40, 56)
    with torch.no_grad():
        ref = R.dncnn_forward(x, sd, depth=6)
        out = m.to(dev)(x.to(dev), 0.1)
    assert rel_err(out, ref) < 3e-2
