"""The TMA convolution kernels on two devices in one process: each device needs its own shared-memory opt-in for every
kernel, so the same layer run first on cuda:0 and then on cuda:1 must launch on both and give the same result."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _layers(dev):
    from deepinv_b200 import ops
    from deepinv_b200.models.tc_engine import _pack3x3, _pack3x3_slab_tc32, _pack_down_tc32

    gen = torch.Generator().manual_seed(7)
    x = torch.randn(2, 64, 24, 40, generator=gen)
    w3 = torch.randn(64, 64, 3, 3, generator=gen) / 24
    wd = torch.randn(128, 64, 2, 2, generator=gen) / 16
    xs = ops.nchw_to_split16(x.to(dev), 1)
    slab = ops.split16_to_nchw(ops.conv_tc32_slab(xs, _pack3x3_slab_tc32(w3.to(dev), 1), 64, relu=True))
    down = ops.split16_to_nchw(ops.conv_tc32(xs, _pack_down_tc32(wd.to(dev), 1), 128, kind=1))
    xb = x.to(torch.bfloat16).permute(0, 2, 3, 1).contiguous()
    bf16 = ops.conv3x3_bf16(xb.to(dev), _pack3x3(w3.to(dev)), relu=True)
    torch.cuda.synchronize(dev)
    return [t.cpu() for t in (slab, down, bf16)]


def test_conv_layers_on_two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    first = _layers(torch.device("cuda:0"))
    second = _layers(torch.device("cuda:1"))
    for a, b in zip(first, second):
        assert torch.equal(a, b)
