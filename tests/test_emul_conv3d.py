"""The CUDA-core kernels of DRUNet(dim=3) on the host emulation (tests/emul): the fp32 3-D convolutions (`dinvk_conv3d_f32`: 3x3x3,
2x2x2 stride 2 and its transpose, with the x + xadd / ReLU / residual / bias fusions) and the split-operand path's 3-D head and
tail (`dinvk_conv3d_tc32_head` / `_tail`), against torch's conv3d in fp64 — the layers of deepinv/models/drunet.py built with
Conv3d / ConvTranspose3d.  Also the weight packing of the 3-D tensor-core engine, restated from the packed matrices, and the
host-side rules of `DRUNet(dim=3)`.  The wgmma layers need an H100 (tests/test_gpu_drunet3d.py)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from emul_util import emul_lib, ptr

CH = {0: 16, 1: 32}
WORD = {0: torch.float32, 1: torch.float16}


def conv3d(x, w, kind, bias=None, xadd=None, res=None, relu=False):
    B, Cin, D, H, W = x.shape
    cout = w.shape[1] if kind == 2 else w.shape[0]
    f = {0: lambda s: s, 1: lambda s: s // 2, 2: lambda s: 2 * s}[kind]
    out = torch.zeros(B, cout, f(D), f(H), f(W))
    rc = emul_lib().dinvk_conv3d_f32(ptr(x.contiguous()), ptr(xadd), ptr(w.contiguous()), ptr(bias), ptr(res), ptr(out), B, Cin, cout,
                                     D, H, W, kind, int(relu), None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def ref3d(x, w, kind, bias=None, xadd=None, res=None, relu=False):
    xi = x.double() if xadd is None else x.double() + xadd.double()
    b = None if bias is None else bias.double()
    if kind == 0:
        y = F.conv3d(xi, w.double(), b, padding=1)
    elif kind == 1:
        y = F.conv3d(xi, w.double(), b, stride=2)
    else:
        y = F.conv_transpose3d(xi, w.double(), b, stride=2)
    if relu:
        y = F.relu(y)
    return y if res is None else y + res.double()


@pytest.mark.parametrize("shape", [(1, 3, 5, 9, 35), (2, 1, 4, 8, 33), (1, 4, 1, 7, 6)])
@pytest.mark.parametrize("fusion", ["plain", "relu_bias", "xadd_res"])
def test_conv3x3x3_f32(shape, fusion):
    """ragged 8 x 32 tiles in H and W, odd D / H / W, D = 1 (only the middle plane of the filter meets the volume), 9 input
    channels (a partial 8-channel step) and 40 output channels (a partial 32-channel CTA)"""
    B, D, H, W = shape[0], shape[2], shape[3], shape[4]
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(B, 9, D, H, W, generator=g)
    w = torch.randn(40, 9, 3, 3, 3, generator=g) / 10
    kw = {}
    if fusion == "relu_bias":
        kw = dict(bias=torch.randn(40, generator=g), relu=True)
    elif fusion == "xadd_res":
        kw = dict(xadd=torch.randn(B, 9, D, H, W, generator=g), res=torch.randn(B, 40, D, H, W, generator=g))
    assert rel_err(conv3d(x, w, 0, **kw).double(), ref3d(x, w, 0, **kw)) < 1e-6


@pytest.mark.parametrize("kind", [1, 2])
@pytest.mark.parametrize("shape", [(2, 4, 6, 10), (1, 2, 2, 2), (1, 6, 4, 34)])
def test_conv2x2x2_f32(kind, shape):
    """both 2x2x2 layers with ragged 64 x 32 GEMM tiles; xadd (the U-Net skip) on the transposed one, residual + ReLU + bias"""
    B, D, H, W = shape
    g = torch.Generator().manual_seed(10 * kind + D)
    cin, cout = 12, 20
    x = torch.randn(B, cin, D, H, W, generator=g)
    w = torch.randn(cin, cout, 2, 2, 2, generator=g) / 4 if kind == 2 else torch.randn(cout, cin, 2, 2, 2, generator=g) / 4
    f = (lambda s: s // 2) if kind == 1 else (lambda s: 2 * s)
    kw = dict(bias=torch.randn(cout, generator=g), relu=True, res=torch.randn(B, cout, f(D), f(H), f(W), generator=g))
    if kind == 2:
        kw["xadd"] = torch.randn(B, cin, D, H, W, generator=g)
    assert rel_err(conv3d(x, w, kind, **kw).double(), ref3d(x, w, kind, **kw)) < 1e-6


def test_conv3d_f32_argument_errors_and_empty_batch():
    lib = emul_lib()
    x, w, out = torch.zeros(64), torch.zeros(64), torch.zeros(64)
    assert lib.dinvk_conv3d_f32(ptr(x), None, ptr(w), None, None, ptr(out), 1, 1, 1, 2, 2, 2, 3, 0, None) != 0
    assert b"kind" in lib.dinvk_last_error()
    assert lib.dinvk_conv3d_f32(ptr(x), None, ptr(w), None, None, ptr(out), 1, 1, 1, 3, 2, 2, 1, 0, None) != 0
    assert b"even" in lib.dinvk_last_error()
    assert lib.dinvk_conv3d_f32(ptr(x), None, ptr(w), None, None, ptr(out), 1, 64, 64, 1 << 20, 1 << 20, 1 << 20, 0, 0, None) != 0
    assert b"too large" in lib.dinvk_last_error()
    n0 = int(lib.dinvk_launch_count())
    assert lib.dinvk_conv3d_f32(ptr(x), None, ptr(w), None, None, ptr(out), 0, 1, 1, 2, 2, 2, 0, 0, None) == 0
    assert int(lib.dinvk_launch_count()) == n0   # the empty batch launches nothing


# ---- split-operand head / tail (CUDA cores) --------------------------------------------------------------------------------
def from_split3d(t, fmt):
    B, D, H, W, nb = t.shape[:5]
    out = torch.zeros(B, nb * CH[fmt], D, H, W)
    rc = emul_lib().dinvk_split16_to_nchw(ptr(t), ptr(out), B, nb * CH[fmt], D * H, W, fmt, None)   # H' = D * H
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def to_split3d(x, fmt):
    B, C, D, H, W = x.shape
    out = torch.zeros(B, D, H, W, C // CH[fmt], 2, CH[fmt], dtype=WORD[fmt])
    rc = emul_lib().dinvk_nchw_to_split16(ptr(x.contiguous()), ptr(out), B, C, D * H, W, fmt, None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def head3d(x, w, fmt, bias=None, fill=None, relu=False, flag=None):
    B, C, D, H, W = x.shape
    cout = w.shape[0]
    out = torch.zeros(B, D, H, W, cout // CH[fmt], 2, CH[fmt], dtype=WORD[fmt])
    rc = emul_lib().dinvk_conv3d_tc32_head(ptr(x.contiguous()), ptr(w.contiguous()), ptr(bias), ptr(out), B, C, D, H, W, cout, 0.0,
                                           ptr(fill), int(fill is not None), int(relu), fmt, ptr(flag), None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def tail3d(t, w, fmt, bias=None, add=None, flag=None):
    B, D, H, W, nb = t.shape[:5]
    cout = w.shape[0]
    out = torch.zeros(B, cout, D, H, W)
    rc = emul_lib().dinvk_conv3d_tc32_tail(ptr(t), ptr(w.contiguous()), ptr(bias), ptr(add), ptr(out), B, D, H, W, nb * CH[fmt], cout,
                                           fmt, ptr(flag), None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("ct,cout,shape", [(3, 64, (2, 3, 5, 7)), (2, 128, (1, 1, 4, 9)), (1, 64, (1, 4, 3, 3))])
def test_head3d(fmt, ct, cout, shape):
    """27 taps from <= 4 NCDHW channels, bias + ReLU; Cout = 128 stages its weights in two 64-channel rounds; the last input
    channel as DRUNet's per-sample noise map (zero outside the volume like every padded channel)"""
    B, D, H, W = shape
    g = torch.Generator().manual_seed(ct + 7 * fmt)
    x = torch.randn(B, ct, D, H, W, generator=g)
    w = torch.randn(cout, ct, 3, 3, 3, generator=g) / 8
    b = torch.randn(cout, generator=g)
    out = from_split3d(head3d(x, w, fmt, bias=b, relu=True), fmt)
    assert rel_err(out.double(), F.relu(F.conv3d(x.double(), w.double(), b.double(), padding=1))) < 1e-6
    if ct >= 2:
        sig = torch.rand(B, generator=g)
        out = from_split3d(head3d(x[:, :ct - 1].contiguous(), w, fmt, fill=sig), fmt)
        xf = torch.cat([x[:, :ct - 1], sig.view(B, 1, 1, 1, 1).expand(B, 1, D, H, W)], 1)
        assert rel_err(out.double(), F.conv3d(xf.double(), w.double(), padding=1)) < 1e-6


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("cin,cout,shape", [(64, 2, (1, 3, 9, 35)), (128, 3, (2, 2, 5, 6)), (64, 1, (1, 1, 8, 32))])
def test_tail3d(fmt, cin, cout, shape):
    """ragged 32 x 8 tiles, two 64-channel chunks at Cin = 128, D = 1; + bias + the NCDHW addend; a raised flag answers NaN"""
    B, D, H, W = shape
    g = torch.Generator().manual_seed(cin + cout + fmt)
    ts = to_split3d(torch.randn(B, cin, D, H, W, generator=g), fmt)
    w = torch.randn(cout, cin, 3, 3, 3, generator=g) / 40
    b = torch.randn(cout, generator=g)
    add = torch.randn(B, cout, D, H, W, generator=g)
    ref = F.conv3d(from_split3d(ts, fmt).double(), w.double(), b.double(), padding=1) + add.double()
    assert rel_err(tail3d(ts, w, fmt, bias=b, add=add).double(), ref) < 1e-6
    assert torch.isnan(tail3d(ts, w, fmt, flag=torch.ones(1, dtype=torch.int32))).all()


def test_head3d_fp16_overflow_raises_the_flag():
    x = torch.full((1, 1, 2, 3, 4), 3.0e5)
    w = torch.ones(64, 1, 3, 3, 3)
    flag = torch.zeros(1, dtype=torch.int32)
    head3d(x, w, 1, flag=flag)
    assert int(flag) == 1
    flag.zero_()
    head3d(x * 1e-3, w, 1, flag=flag)
    assert int(flag) == 0


def test_head_tail_errors_and_empty_batch():
    lib = emul_lib()
    buf = torch.zeros(1 << 12)
    assert lib.dinvk_conv3d_tc32_head(ptr(buf), ptr(buf), None, ptr(buf), 1, 4, 2, 2, 2, 64, 0.0, None, 1, 0, 0, None, None) != 0
    assert lib.dinvk_conv3d_tc32_tail(ptr(buf), ptr(buf), None, None, ptr(buf), 1, 2, 2, 2, 64, 5, 0, None, None) != 0
    assert lib.dinvk_conv3d_tc32_tail(ptr(buf), ptr(buf), None, None, ptr(buf), 1, 2, 2, 2, 48, 2, 1, None, None) != 0   # not a CH multiple
    assert lib.dinvk_conv3d_tc32_head(ptr(buf), ptr(buf), None, ptr(buf), 1, 1, 1 << 20, 1 << 20, 1 << 20, 64, 0.0, None, 0, 0, 0,
                                      None, None) != 0
    assert b"too large" in lib.dinvk_last_error()
    n0 = int(lib.dinvk_launch_count())
    assert lib.dinvk_conv3d_tc32_head(ptr(buf), ptr(buf), None, ptr(buf), 0, 1, 2, 2, 2, 64, 0.0, None, 0, 0, 0, None, None) == 0
    assert lib.dinvk_conv3d_tc32_tail(ptr(buf), ptr(buf), None, None, ptr(buf), 0, 2, 2, 2, 64, 2, 0, None, None) == 0
    assert int(lib.dinvk_launch_count()) == n0


# ---- weight packing of the 3-D engine (pure torch) -------------------------------------------------------------------------
def _unpack(p, fmt, rows):
    """(2*rows, K) packed [hi; lo] per 64 rows -> (rows, K) fp64 hi + lo"""
    K = p.shape[1]
    q = p.double().view(rows // 64, 2, 64, K)
    return (q[:, 0] + q[:, 1] * (2.0 ** -11 if fmt == 1 else 1.0)).reshape(rows, K)


@pytest.mark.parametrize("fmt", [0, 1])
def test_packing_restates_conv3d(fmt):
    from deepinv_b200.models.tc_engine import _pack3x3x3_tc32, _pack_down3d_tc32, _pack_up3d_tc32

    g = torch.Generator().manual_seed(fmt)
    cin, cout = 64, 128
    x = torch.randn(1, cin, 4, 6, 6, generator=g, dtype=torch.float64)
    # 3x3x3: out[co, v] = sum_{tap, c} Wk[co, tap * Cin + c] * x[c, v + tap - 1]
    w = torch.randn(cout, cin, 3, 3, 3, generator=g) / 20
    wk = _unpack(_pack3x3x3_tc32(w, fmt), fmt, cout)
    xp = F.pad(x, (1, 1, 1, 1, 1, 1))
    cols = torch.stack([xp[0, :, kz:kz + 4, ky:ky + 6, kx:kx + 6] for kz in range(3) for ky in range(3) for kx in range(3)])
    out = (wk @ cols.reshape(27 * cin, -1)).view(1, cout, 4, 6, 6)
    assert rel_err(out, F.conv3d(x, w.double(), padding=1)) < 1e-6
    # 2x2x2 down: k = (dz*4+dy*2+dx)*Cin + c
    wd = torch.randn(cout, cin, 2, 2, 2, generator=g) / 10
    wk = _unpack(_pack_down3d_tc32(wd, fmt), fmt, cout)
    cols = torch.stack([x[0, :, dz::2, dy::2, dx::2] for dz in range(2) for dy in range(2) for dx in range(2)])
    out = (wk @ cols.reshape(8 * cin, -1)).view(1, cout, 2, 3, 3)
    assert rel_err(out, F.conv3d(x, wd.double(), stride=2)) < 1e-6
    # 2x2x2 up: row = (dz*4+dy*2+dx)*Cout + co
    wu = torch.randn(cin, cout, 2, 2, 2, generator=g) / 10
    wk = _unpack(_pack_up3d_tc32(wu, fmt), fmt, 8 * cout)
    prod = (wk @ x[0].reshape(cin, -1)).view(2, 2, 2, cout, 4, 6, 6)
    out = prod.permute(3, 4, 0, 5, 1, 6, 2).reshape(1, cout, 8, 12, 12)
    assert rel_err(out, F.conv_transpose3d(x, wu.double(), stride=2)) < 1e-6


# ---- DRUNet(dim=3) host rules ----------------------------------------------------------------------------------------------
def test_drunet3d_modules_dims_and_errors():
    import deepinv_b200 as dinv

    m = dinv.models.DRUNet(in_channels=2, out_channels=2, nc=(64, 64, 128, 128), nb=1, pretrained=None, dim="3d")
    assert m.dim == 3
    sd = m.state_dict()
    assert tuple(sd["m_head.weight"].shape) == (64, 3, 3, 3, 3)
    assert tuple(sd["m_down1.1.weight"].shape) == (64, 64, 2, 2, 2)
    assert tuple(sd["m_up3.0.weight"].shape) == (128, 128, 2, 2, 2)
    assert tuple(sd["m_tail.weight"].shape) == (2, 64, 3, 3, 3)
    for d in (3, "3", "3D"):
        assert dinv.models.DRUNet(nc=(64, 64, 64, 64), nb=1, pretrained=None, dim=d).dim == 3
    for d in (4, "4d", 1.5):
        with pytest.raises(ValueError):
            dinv.models.DRUNet(pretrained=None, dim=d)
    with pytest.raises(RuntimeError):
        dinv.models.DRUNet(pretrained="download_2d", dim=3)
    with pytest.raises(NotImplementedError):
        dinv.models.DRUNet(nc=(64, 64, 64, 64), nb=1, pretrained=None, dim=3, precision="bf16")
    x = torch.zeros(1, 2, 8, 8, 8)
    with pytest.raises(ValueError):
        m(x, torch.ones(1, 1, 1, 1))       # the 2-D shape of a per-sample sigma
    with pytest.raises(NotImplementedError, match="test_onesplit"):
        m.eval()(torch.zeros(1, 2, 64, 70, 66), 0.1)   # in training mode the reference pads instead
    with pytest.raises(NotImplementedError):
        m(x.requires_grad_(), 0.1)         # no gradients through the 3-D network
