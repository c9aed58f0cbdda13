"""`crop` of the MRI operators (deepinv/utils/mixins.py:208-247, torchvision's CenterCrop): the centre crop to img_size[-2:], with
an odd height cropped to H + 1 rows and the last row dropped.  CenterCrop zero-pads an input smaller than the crop, so an odd
height equal to the input's own keeps all H rows (and an input smaller than img_size comes back zero-padded to it)."""
import pytest
import torch


def _mixin(img_size):
    from deepinv_b200.physics.mri import MRIMixin

    m = MRIMixin()
    m.img_size = img_size
    return m


def _center_crop(x, ch, cw):
    """torchvision's CenterCrop on (..., h, w), restated: zero-pad to at least (ch, cw) (the smaller half first), then crop at
    int(round((h - ch) / 2)), int(round((w - cw) / 2))"""
    h, w = x.shape[-2:]
    ph, pw = max(ch - h, 0), max(cw - w, 0)
    x = torch.nn.functional.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    h, w = x.shape[-2:]
    t, l = int(round((h - ch) / 2.0)), int(round((w - cw) / 2.0))
    return x[..., t: t + ch, l: l + cw]


@pytest.mark.parametrize("img,shape", [((2, 17, 11), (1, 2, 17, 11)), ((2, 15, 11), (1, 2, 17, 11)), ((2, 16, 12), (1, 2, 20, 14)),
                                       ((2, 15, 11), (2, 2, 20, 14)), ((2, 320, 320), (1, 2, 640, 368)),
                                       ((2, 17, 11), (1, 2, 16, 10)), ((2, 5, 17, 11), (2, 2, 5, 17, 11))])
def test_crop(img, shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(0))
    got = _mixin(img).crop(x)
    H, W = img[-2:]
    want = _center_crop(x, H + 1, W)[..., :-1, :] if H % 2 else _center_crop(x, H, W)
    assert got.shape == (*shape[:-2], H, W) and torch.equal(got, want)


def test_odd_height_equal_to_the_input_keeps_every_row():
    x = torch.randn(2, 2, 17, 11, generator=torch.Generator().manual_seed(1))
    assert torch.equal(_mixin((2, 17, 11)).crop(x), x)
