"""The CUDA-core kernels of the fp32-grade denoiser path on the host emulation (tests/emul): network head (NCHW fp32 -> split
layout, `head64_tc32_kernel` with lanes = output channels and the thread-per-pixel first version), network tail (split layout ->
NCHW fp32, `tail64_tc32_kernel` with lanes = input channels + the transposing shuffle reduction, and the shared-memory first
version) and the layout converters, for both split formats (fmt 0: tf32 words, fmt 1: fp16 words).  Checked against
torch's conv2d in fp64 — the layers deepinv/models/drunet.py:150-176 (m_head / m_tail) and dncnn.py:94-131 (in_conv /
out_conv + x) put at the ends of the networks.  The wgmma body layers need an H100 (tests/test_gpu_tc32.py)."""
import ctypes as C
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from emul_util import emul_lib, ptr

CH = {0: 16, 1: 32}
WORD = {0: torch.float32, 1: torch.float16}


def to_split(x, fmt):
    B, Cc, H, W = x.shape
    out = torch.zeros(B, H, W, Cc // CH[fmt], 2, CH[fmt], dtype=WORD[fmt])
    rc = emul_lib().dinvk_nchw_to_split16(ptr(x.contiguous()), ptr(out), B, Cc, H, W, fmt, None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def from_split(t, fmt):
    B, H, W, nb = t.shape[:4]
    out = torch.zeros(B, nb * CH[fmt], H, W)
    rc = emul_lib().dinvk_split16_to_nchw(ptr(t), ptr(out), B, nb * CH[fmt], H, W, fmt, None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def head(x, w, fmt, bias=None, fill=None, relu=False, flag=None):
    B, Cc, H, W = x.shape
    cout = w.shape[0]
    out = torch.zeros(B, H, W, cout // CH[fmt], 2, CH[fmt], dtype=WORD[fmt])
    rc = emul_lib().dinvk_conv_tc32_head(ptr(x.contiguous()), ptr(w.contiguous()), ptr(bias), ptr(out), B, Cc, H, W, cout, 0.0,
                                         ptr(fill), int(fill is not None), int(relu), fmt, ptr(flag), None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


def tail(t, w, fmt, bias=None, add=None, flag=None):
    B, H, W, nb = t.shape[:4]
    cout = w.shape[0]
    out = torch.zeros(B, cout, H, W)
    rc = emul_lib().dinvk_conv_tc32_tail(ptr(t), ptr(w.contiguous()), ptr(bias), ptr(add), ptr(out), B, H, W, nb * CH[fmt], cout, fmt,
                                         ptr(flag), None)
    assert rc == 0, emul_lib().dinvk_last_error()
    return out


@pytest.mark.parametrize("fmt", [0, 1])
def test_converters_roundtrip(fmt):
    gen = torch.Generator().manual_seed(fmt)
    x = torch.randn(2, 64, 5, 7, generator=gen)
    back = from_split(to_split(x, fmt), fmt)
    if fmt == 0:
        assert torch.equal(back, x)                       # tf32 split: hi + lo == v bit for bit
    else:
        assert rel_err(back.double(), x.double()) < 2.0 ** -21


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("ct,shape", [(3, (2, 9, 40)), (2, (1, 5, 70)), (1, (1, 4, 33)), (4, (1, 3, 32))])
def test_head_lanes_are_channels(fmt, ct, shape):
    """Cout = 64: two rows x 32 pixels per warp, odd heights / partial and multiple row segments; bias + ReLU; per-sample fill channel"""
    B, H, W = shape
    gen = torch.Generator().manual_seed(10 * ct + fmt)
    x = torch.randn(B, ct, H, W, generator=gen)
    w = torch.randn(64, ct, 3, 3, generator=gen) / 5
    b = torch.randn(64, generator=gen)
    out = from_split(head(x, w, fmt, bias=b, relu=True), fmt)
    assert rel_err(out.double(), F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1))) < 1e-6
    if ct >= 2:   # the last input channel as DRUNet's constant noise map (zero outside the image like every padded channel)
        sig = torch.rand(B, generator=gen)
        out = from_split(head(x[:, :ct - 1].contiguous(), w, fmt, fill=sig), fmt)
        xf = torch.cat([x[:, :ct - 1], sig.view(B, 1, 1, 1).expand(B, 1, H, W)], 1)
        assert rel_err(out.double(), F.conv2d(xf.double(), w.double(), padding=1)) < 1e-6


@pytest.mark.parametrize("fmt", [0, 1])
def test_head_other_widths_use_the_thread_per_pixel_kernel(fmt):
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(1, 3, 6, 11, generator=gen)
    w = torch.randn(128, 3, 3, 3, generator=gen) / 5
    out = from_split(head(x, w, fmt), fmt)
    assert rel_err(out.double(), F.conv2d(x.double(), w.double(), padding=1)) < 1e-6


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("cout", [1, 2, 3, 4])
@pytest.mark.parametrize("shape", [(2, 7, 19), (1, 37, 9), (1, 70, 10)])
def test_tail_lanes_are_channels(fmt, cout, shape):
    """Cin = 64: strips of 16 / 8 / 4 columns x 32-row chunks (one partial chunk, two chunks, three chunks), + bias + the NCHW addend"""
    B, H, W = shape
    gen = torch.Generator().manual_seed(100 * cout + fmt)
    t = torch.randn(B, 64, H, W, generator=gen)
    w = torch.randn(cout, 64, 3, 3, generator=gen) / 24
    b = torch.randn(cout, generator=gen)
    add = torch.randn(B, cout, H, W, generator=gen)
    ts = to_split(t, fmt)
    out = tail(ts, w, fmt, bias=b, add=add)
    ref = F.conv2d(from_split(ts, fmt).double(), w.double(), b.double(), padding=1) + add.double()
    assert rel_err(out.double(), ref) < 1e-6


@pytest.mark.parametrize("fmt", [0, 1])
def test_tail_old_kernel_and_overflow_flag(fmt):
    """Cin = 128 runs the shared-memory first version; a raised overflow flag turns the whole output into NaN"""
    gen = torch.Generator().manual_seed(5)
    t = torch.randn(1, 128, 6, 10, generator=gen)
    w = torch.randn(2, 128, 3, 3, generator=gen) / 34
    ts = to_split(t, fmt)
    ref = F.conv2d(from_split(ts, fmt).double(), w.double(), padding=1)
    assert rel_err(tail(ts, w, fmt).double(), ref) < 1e-6
    flag = torch.ones(1, dtype=torch.int32)
    t64 = to_split(torch.randn(1, 64, 4, 8, generator=gen), fmt)
    assert torch.isnan(tail(t64, torch.randn(2, 64, 3, 3, generator=gen), fmt, flag=flag)).all()


def test_head_fp16_overflow_raises_the_flag():
    x = torch.full((1, 1, 4, 32), 3.0e5)
    w = torch.ones(64, 1, 3, 3)
    flag = torch.zeros(1, dtype=torch.int32)
    head(x, w, 1, flag=flag)
    assert int(flag) == 1
    flag.zero_()
    head(x * 1e-3, w, 1, flag=flag)
    assert int(flag) == 0


# ---------------------------------------------------------------------------------------------------------------------------
# The package's fp32-grade denoiser ENGINES on the host: tc_engine.py (weight packing, ResBlock / skip wiring, per-call overflow
# flag) driving the emulated head / tail kernels and the scalar model of the tensor-core layers (tests/emul/conv_tc32_model.cu),
# against the oracle's fp32 networks (drunet.py:200-263, dncnn.py:116-140).  What this pins is the HOST logic; the wgmma kernels
# behind the same ABI are compared with the same oracle on the H100 (tests/test_gpu_tc32.py).
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def emul_backend(monkeypatch):
    from deepinv_b200 import ops

    lib = emul_lib()

    def check(rc):
        assert rc == 0, lib.dinvk_last_error()

    monkeypatch.setattr(ops, "_require_cuda", lambda *ts: torch.device("cpu"))
    monkeypatch.setattr(ops, "_stream", lambda dev: None)
    monkeypatch.setattr(ops, "get_lib", lambda: lib)
    monkeypatch.setattr(ops, "check", check)
    ops._ws_cache.clear()
    yield
    ops._ws_cache.clear()


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_drunet_engine_on_the_model(precision, emul_backend):
    import deepinv_b200 as dinv
    from deepinv_b200.models.tc_engine import tc_overflow
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, nb=1, pretrained=None, precision=precision).eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(1, 2, 16, 16)
    with torch.no_grad():
        out = m(x, 0.07)
        ref = R.drunet_forward(x, 0.07, sd, nb=1)
        assert rel_err(out, ref) < 1e-5 and not tc_overflow(m)
        per = m(x, torch.tensor([0.07]))                  # per-sample noise level: the head's fill channel from a device vector
        assert rel_err(per, ref) < 1e-5
        if precision == "tc32h":                          # out-of-range input: that call answers NaN, the next one is served normally
            assert torch.isnan(m(x * 3e6, 0.07)).all() and tc_overflow(m)
            assert torch.equal(m(x, 0.07), out) and not tc_overflow(m)


@pytest.mark.parametrize("precision", ["tc32", "tc32h"])
def test_dncnn_engine_on_the_model(precision, emul_backend):
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(1)
    m = dinv.models.DnCNN(in_channels=1, out_channels=1, depth=4, nf=64, pretrained=None, precision=precision).eval()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    x = torch.randn(2, 1, 9, 12)
    with torch.no_grad():
        assert rel_err(m(x, 0.1), R.dncnn_forward(x, sd, depth=4)) < 1e-5


def test_pnp_pgd_loop_with_the_tc32h_engine(emul_backend):
    """the benchmark's loop in miniature on the host: PnP-PGD on single-coil MRI (emulated spectral kernels) with the tc32h DRUNet
    engine (emulated head / tail + model layers), 3 iterations, against the oracle's loop (pgd.py:137-168)"""
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PGD, PnP
    from oracle import ref_ops as R

    torch.manual_seed(0)
    B, H, W = 1, 16, 16
    x = torch.randn(B, 2, H, W)
    cols = (torch.rand(B, 1, 1, W) > 0.6).float()
    cols[..., W // 2 - 2: W // 2 + 2] = 1
    mask = cols.expand(B, 2, H, W).contiguous()
    den = dinv.models.DRUNet(in_channels=2, out_channels=2, nb=1, pretrained=None, precision="tc32h").eval()
    sd = {k: v.detach().clone() for k, v in den.state_dict().items()}
    y = R.mri_A(x, mask)
    with torch.no_grad():
        ref = R.pgd(y, lambda v: R.mri_A(v, mask), lambda v: R.mri_At(v, mask), lambda v, s: R.drunet_forward(v, s, sd, nb=1), 1.0, 0.05, 3)
        physics = dinv.physics.MRI(mask=mask, img_size=(2, H, W), device="cpu")
        algo = PGD(data_fidelity=L2(), prior=PnP(den), stepsize=1.0, sigma_denoiser=0.05, max_iter=3, early_stop=False)
        out = algo(y, physics)
    assert rel_err(out, ref) < 1e-5
