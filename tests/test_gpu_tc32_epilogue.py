"""GPU tests of the split-operand convolutions' epilogue (csrc/conv_tc32.cu) on persistent launches in which every CTA
runs several work items and the CTAs run unequal numbers of them.  A result may not depend on which CTA computed a tile or
on what that CTA computed before: each layer must equal, bit for bit, the same images run one per launch, and must stay
within 2e-6 of an fp64 evaluation."""
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


def _to_split(x, dev, fmt):
    from deepinv_b200 import ops

    return ops.nchw_to_split16(x.to(dev), fmt)


def _from_split(t):
    from deepinv_b200 import ops

    return ops.split16_to_nchw(t).cpu()


def _batch(dev, items_per_image):
    """smallest batch with at least two work items per SM whose item count is not a multiple of the SM count"""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    B = 2 * sms // items_per_image + 1
    while (B * items_per_image) % sms == 0:
        B += 1
    assert B * items_per_image >= 2 * sms
    return B


def _per_image(fn, *tensors):
    """fn run on one image per launch (then every CTA runs at most one work item), results concatenated"""
    return torch.cat([fn(*(t[i:i + 1] if t is not None else None for t in tensors)) for i in range(tensors[0].shape[0])])


def _cdiv(a, b):
    return -(-a // b)


@pytest.mark.parametrize("cin,cout,H,W", [(64, 64, 40, 36), (64, 128, 24, 44), (128, 192, 20, 18)])
@pytest.mark.parametrize("fmt", [0, 1])
def test_slab_multi_item(cin, cout, H, W, fmt, dev):
    """3x3 slab kernel (16 x 16-pixel tiles): partial tiles in both dimensions, N tiles at offsets 0 / 64 / 128 of a pixel
    row, bias + ReLU + res + res2"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3_slab_tc32

    B = _batch(dev, _cdiv(H, 16) * _cdiv(W, 16) * (cout // 64))
    gen = torch.Generator().manual_seed(11)
    x = torch.randn(B, cin, H, W, generator=gen).abs()
    w = torch.randn(cout, cin, 3, 3, generator=gen) / (3 * cin ** 0.5)
    r1, r2 = torch.randn(B, cout, H, W, generator=gen), torch.randn(B, cout, H, W, generator=gen)
    bias = torch.randn(cout, generator=gen)
    wp, bd = _pack3x3_slab_tc32(w.to(dev), fmt), bias.to(dev)
    xs, rs1, rs2 = _to_split(x, dev, fmt), _to_split(r1, dev, fmt), _to_split(r2, dev, fmt)

    def run(xx, a, b):
        return ops.conv_tc32_slab(xx, wp, cout, bias=bd, res=a, res2=b, relu=True)

    out = run(xs, rs1, rs2)
    ref = F.relu(F.conv2d(x.double(), w.double(), bias.double(), padding=1)) + r1.double() + r2.double()
    assert rel_err(_from_split(out).double(), ref) < 2e-6
    assert torch.equal(out, _per_image(run, xs, rs1, rs2))


@pytest.mark.parametrize("fmt", [0, 1])
def test_per_tap_down_multi_item(fmt, dev):
    """2x2 stride-2 layer (kind 1) on the per-tap kernel (16 x 8-pixel tiles), partial tiles in both dimensions"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack_down_tc32

    cin, cout, H, W = 64, 128, 44, 40
    B = _batch(dev, _cdiv(H // 2, 8) * _cdiv(W // 2, 16) * (cout // 64))
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(B, cin, H, W, generator=gen)
    wd = torch.randn(cout, cin, 2, 2, generator=gen) / (2 * cin ** 0.5)
    wp = _pack_down_tc32(wd.to(dev), fmt)
    xs = _to_split(x, dev, fmt)

    def run(xx):
        return ops.conv_tc32(xx, wp, cout, kind=1)

    out = run(xs)
    assert rel_err(_from_split(out).double(), F.conv2d(x.double(), wd.double(), stride=2)) < 2e-6
    assert torch.equal(out, _per_image(run, xs))


@pytest.mark.parametrize("fmt", [0, 1])
def test_per_tap_up_multi_item(fmt, dev):
    """transposed 2x2 stride-2 layer (kind 2): every N tile scatters to its own output sub-pixel"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack_up_tc32

    cin, cout, H, W = 128, 64, 12, 20   # input grid; output (2H, 2W)
    B = _batch(dev, _cdiv(H, 8) * _cdiv(W, 16) * (4 * cout // 64))
    gen = torch.Generator().manual_seed(13)
    x = torch.randn(B, cin, H, W, generator=gen)
    wt = torch.randn(cin, cout, 2, 2, generator=gen) / (cin ** 0.5)   # ConvTranspose2d(cin -> cout) weight
    wp = _pack_up_tc32(wt.to(dev), fmt)
    xs = _to_split(x, dev, fmt)

    def run(xx):
        return ops.conv_tc32(xx, wp, cout, kind=2)

    out = run(xs)
    assert out.shape[:3] == (B, 2 * H, 2 * W)
    assert rel_err(_from_split(out).double(), F.conv_transpose2d(x.double(), wt.double(), stride=2)) < 2e-6
    assert torch.equal(out, _per_image(run, xs))


def test_overflow_in_last_work_item(dev):
    """fp16 format: the only output beyond the fp16 range is in the last work item of the launch (the bottom-right tile of
    the last image), which is the last item of its CTA; the flag is raised all the same"""
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3_slab_tc32

    C, H, W = 64, 40, 36
    B = _batch(dev, _cdiv(H, 16) * _cdiv(W, 16))
    gen = torch.Generator().manual_seed(14)
    x = torch.rand(B, C, H, W, generator=gen)
    w = torch.randn(C, C, 3, 3, generator=gen) / (3 * C ** 0.5)
    r = torch.zeros(B, C, H, W)
    wp, xs = _pack3x3_slab_tc32(w.to(dev), 1), _to_split(x, dev, 1)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.conv_tc32_slab(xs, wp, C, res=_to_split(r, dev, 1), res2=_to_split(r, dev, 1), flag=flag)
    assert int(flag.item()) == 0
    r[-1, 5, H - 1, W - 1] = 64000.0   # res + res2 = 128000: only this output element leaves the range
    rs = _to_split(r, dev, 1)
    ops.conv_tc32_slab(xs, wp, C, res=rs, res2=rs, flag=flag)
    assert int(flag.item()) == 1
