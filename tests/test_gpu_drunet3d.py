"""DRUNet(dim=3) on the H100: every 3-D layer kind of the split-operand wgmma path (`dinvk_conv3d_tc32`, the per-tap kernel with
its depth axis) at DRUNet widths, both split formats and drain windows 1 and 2, against fp64 conv3d / conv_transpose3d; the 3-D
CUDA-core fp32 layers; the whole network at fp32 / tc32 / tc32h against an fp64 restatement of the reference's Conv3d network
(deepinv/models/drunet.py); run-to-run bitwise; the per-call fp16 overflow flag; argument errors; PnP-PGD on 3-D MRI."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from drunet3d_ref64 import drunet3d_ref64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def to_split3d(x, dev, fmt):
    from deepinv_b200 import ops

    B, C, D, H, W = x.shape
    t = ops.nchw_to_split16(x.to(dev).reshape(B, C, D * H, W), fmt)   # the 2-D converter with H' = D * H
    return t.view(B, D, H, W, *t.shape[3:])


def from_split3d(t):
    from deepinv_b200 import ops

    B, D, H, W = t.shape[:4]
    out = ops.split16_to_nchw(t.reshape(B, D * H, W, *t.shape[4:])).cpu()
    return out.view(B, -1, D, H, W)


LAYERS = [  # (kind, Cin, Cout, (B, D, H, W)): sizes cross the 16 x 8 tile edges in H and W, several depth planes
    (0, 64, 64, (1, 3, 20, 35)), (0, 128, 128, (2, 2, 9, 17)), (0, 256, 256, (1, 3, 8, 16)), (0, 512, 512, (1, 2, 5, 9)),
    (1, 64, 128, (1, 4, 18, 34)), (1, 128, 256, (2, 2, 10, 20)), (1, 256, 512, (1, 2, 8, 18)),
    (2, 512, 256, (1, 2, 5, 9)), (2, 256, 128, (1, 2, 9, 10)), (2, 128, 64, (1, 3, 9, 17)),
]


@pytest.mark.parametrize("layer", LAYERS, ids=lambda l: f"k{l[0]}_{l[1]}to{l[2]}")
@pytest.mark.parametrize("window", [1, 2])
@pytest.mark.parametrize("fmt", [0, 1])
def test_conv3d_tc32_layers(layer, window, fmt, dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3x3_tc32, _pack_down3d_tc32, _pack_up3d_tc32

    kind, cin, cout, (B, D, H, W) = layer
    g = torch.Generator().manual_seed(kind * 1000 + cin + fmt)
    x = torch.randn(B, cin, D, H, W, generator=g).abs()
    xs = to_split3d(x, dev, fmt)
    xr = from_split3d(xs).double()   # the operand as the kernel holds it (exact for tf32 words)
    if kind == 0:
        w = torch.randn(cout, cin, 3, 3, 3, generator=g) / (5 * cin ** 0.5)
        bias = torch.randn(cout, generator=g)
        r1, r2 = torch.randn(B, cout, D, H, W, generator=g), torch.randn(B, cout, D, H, W, generator=g)
        out = from_split3d(ops.conv3d_tc32(xs, _pack3x3x3_tc32(w.to(dev), fmt), cout, bias=bias.to(dev), res=to_split3d(r1, dev, fmt),
                                           res2=to_split3d(r2, dev, fmt), relu=True, window=window))
        ref = F.relu(F.conv3d(xr, w.double(), bias.double(), padding=1)) + from_split3d(to_split3d(r1, dev, fmt)).double() \
            + from_split3d(to_split3d(r2, dev, fmt)).double()
        assert rel_err(out.double(), ref) < 2e-6
        out = from_split3d(ops.conv3d_tc32(xs, _pack3x3x3_tc32(w.to(dev), fmt), cout, window=window))
        assert rel_err(out.double(), F.conv3d(xr, w.double(), padding=1)) < 2e-6
    elif kind == 1:
        w = torch.randn(cout, cin, 2, 2, 2, generator=g) / (2 * cin ** 0.5)
        out = from_split3d(ops.conv3d_tc32(xs, _pack_down3d_tc32(w.to(dev), fmt), cout, kind=1, window=window))
        assert rel_err(out.double(), F.conv3d(xr, w.double(), stride=2)) < 2e-6
    else:
        w = torch.randn(cin, cout, 2, 2, 2, generator=g) / cin ** 0.5
        out = from_split3d(ops.conv3d_tc32(xs, _pack_up3d_tc32(w.to(dev), fmt), cout, kind=2, window=window))
        assert rel_err(out.double(), F.conv_transpose3d(xr, w.double(), stride=2)) < 2e-6


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_conv3d_f32_layers(kind, dev):
    from deepinv_b200 import ops

    g = torch.Generator().manual_seed(kind)
    x = torch.randn(2, 64, 4, 18, 40, generator=g)
    xa = torch.randn(2, 64, 4, 18, 40, generator=g)
    if kind == 0:
        w = torch.randn(64, 64, 3, 3, 3, generator=g) / 40
        ref = F.conv3d((x + xa).double(), w.double(), padding=1)
    elif kind == 1:
        w = torch.randn(128, 64, 2, 2, 2, generator=g) / 20
        ref = F.conv3d((x + xa).double(), w.double(), stride=2)
    else:
        w = torch.randn(64, 32, 2, 2, 2, generator=g) / 20
        ref = F.conv_transpose3d((x + xa).double(), w.double(), stride=2)
    out = ops.conv3d_f32(x.to(dev), w.to(dev), kind=kind, xadd=xa.to(dev)).cpu()
    assert rel_err(out.double(), ref) < 1e-6


# ---- the whole network ---------------------------------------------------------------------------------------------------
def _model(dev, precision, nc=(64, 64, 128, 128), nb=1, ch=2, seed=0):
    import deepinv_b200 as dinv

    torch.manual_seed(seed)
    return dinv.models.DRUNet(in_channels=ch, out_channels=ch, nc=nc, nb=nb, pretrained=None, dim=3, precision=precision).to(dev).eval()


@pytest.mark.parametrize("precision", ["fp32", "tc32", "tc32h"])
@pytest.mark.parametrize("case", ["safe", "padded_c1", "padded_small"])
def test_drunet3d_small_widths(precision, case, dev):
    """a safe shape (32, 32, 40) and the replicate-padded ones (16, 24, 20), (8, 16, 16); C = 1 and 2; scalar, (B,),
    (B, 1, 1, 1, 1) and full-map sigma"""
    ch, shape = {"safe": (2, (2, 32, 32, 40)), "padded_c1": (1, (2, 16, 24, 20)), "padded_small": (2, (1, 8, 16, 16))}[case]
    m = _model(dev, precision, ch=ch)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(3)
    B = shape[0]
    x = torch.randn(B, ch, *shape[1:], generator=g)
    sigmas = [0.05, torch.full((B,), 0.07), torch.full((B, 1, 1, 1, 1), 0.03), 0.1 * torch.rand(B, 1, *shape[1:], generator=g)]
    with torch.no_grad():
        for s in sigmas:
            out = m(x.to(dev), s.to(dev) if torch.is_tensor(s) else s).cpu()
            assert out.shape == x.shape
            xp = x
            sp = s
            if case != "safe":   # the reference's test_pad: replicate padding to a multiple of 16, then a crop
                pad = [(-d) % 16 for d in shape[1:]]
                padding = (0, pad[2], 0, pad[1], 0, pad[0])
                xp = F.pad(x, padding, mode="replicate")
                if torch.is_tensor(s) and s.dim() == 5 and s.shape[2:] == x.shape[2:]:
                    sp = F.pad(s, padding, mode="replicate")
            ref = drunet3d_ref64(xp, sp, sd, nb=1)[..., :shape[1], :shape[2], :shape[3]]
            assert rel_err(out.double(), ref) < 1e-5, (precision, case, s if not torch.is_tensor(s) else tuple(s.shape))


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_drunet3d_full_width_and_bitwise(precision, dev):
    m = _model(dev, precision, nc=(64, 128, 256, 512), nb=2, seed=1)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 2, 32, 32, 32, generator=g).to(dev)
    with torch.no_grad():
        a = m(x, 0.05)
        b = m(x, 0.05)
        ref = drunet3d_ref64(x, 0.05, sd, nb=2)
    assert torch.equal(a, b)
    assert rel_err(a, ref) < 1e-5


def test_drunet3d_overflow_poisons_its_own_call(dev):
    from deepinv_b200.models.tc_engine import tc_overflow

    m = _model(dev, "tc32h")
    x = torch.randn(1, 2, 8, 16, 16, device=dev)
    with torch.no_grad():
        good = m(x, 0.05)
        assert not tc_overflow(m)
        assert torch.isnan(m(x * 3e6, 0.05)).all() and tc_overflow(m)
        assert torch.equal(m(x, 0.05), good) and not tc_overflow(m)


def test_conv3d_tc32_argument_errors(dev):
    from deepinv_b200._lib import get_lib

    lib = get_lib()
    buf = torch.zeros(1 << 16, device=dev)
    p = buf.data_ptr()
    call = lambda B, D, H, W, cin, cout, kind, res=None: lib.dinvk_conv3d_tc32(p, p, None, res, None, p, B, D, H, W, cin, cout, kind, 0, 0, 0,
                                                                                None, None)
    assert call(1, 2, 8, 8, 64, 64, 3) != 0 and b"kind" in lib.dinvk_last_error()
    assert call(1, 3, 8, 8, 64, 64, 1) != 0 and b"even" in lib.dinvk_last_error()
    assert call(1, 2, 8, 8, 48, 64, 0) != 0 and b"Cin" in lib.dinvk_last_error()
    assert call(1, 2, 8, 8, 64, 96, 0) != 0 and b"Cout" in lib.dinvk_last_error()
    assert call(1, 1 << 20, 1 << 20, 1 << 20, 64, 64, 0) != 0 and b"too large" in lib.dinvk_last_error()
    assert call(1, 2, 8, 8, 64, 64, 1, res=p) != 0
    n0 = int(lib.dinvk_launch_count())
    assert call(0, 2, 8, 8, 64, 64, 0) == 0
    assert int(lib.dinvk_launch_count()) == n0


def test_pnp_pgd_mri3d_tc32h(dev):
    """MRI(three_d=True) + PGD(L2(), PnP(DRUNet(dim=3, precision="tc32h"))) against the same loop with the fp64 restatement of
    the denoiser: no torch convolution runs in the library's loop"""
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP

    den = _model(dev, "tc32h")
    sd = {k: v.detach() for k, v in den.state_dict().items()}

    class Ref(torch.nn.Module):
        def forward(self, x, sigma):
            pad = [(-d) % 16 for d in x.shape[2:]]
            xp = F.pad(x, (0, pad[2], 0, pad[1], 0, pad[0]), mode="replicate")
            return drunet3d_ref64(xp, sigma, sd, nb=1)[..., :x.shape[2], :x.shape[3], :x.shape[4]].float()

    g = torch.Generator().manual_seed(5)
    D, H, W = 8, 16, 16
    x = torch.randn(1, 2, D, H, W, generator=g).to(dev)
    mask = (torch.rand(D, H, W, generator=g) > 0.5).float().to(dev)
    phys = dinv.physics.MRI(mask=mask, img_size=(2, D, H, W), three_d=True, device=dev)
    y = phys.A(x)
    with torch.no_grad():
        outs = [PGD(data_fidelity=L2(), prior=PnP(d), stepsize=1.0, sigma_denoiser=0.05, max_iter=4, early_stop=False)(y, phys)
                for d in (den, Ref())]
    assert rel_err(outs[0], outs[1]) < 1e-5
