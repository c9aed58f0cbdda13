"""fp64 restatement of the reference's 3-D DRUNet forward (deepinv/models/drunet.py built with Conv3d / ConvTranspose3d, bias-free)
and the seeded weights of the drunet3d_* golden fixtures (tests/golden/make_golden_drunet3d.py)."""
import numpy as np
import torch
import torch.nn.functional as F


def weights(seed, shapes):
    """the fixtures' deterministic weights for state_dict names / shapes `shapes` (make_golden_drunet3d.weights)"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        s = tuple(shapes[k])
        fan = int(np.prod(s[1:]))
        out[k] = torch.randn(s, generator=g) * (0.5 / fan ** 0.5)
    return out


def wsum(sd):
    ks = sorted(sd)
    return np.array([sum(float(sd[k].double().sum()) for k in ks), sum(float(sd[k].double().pow(2).sum()) for k in ks),
                     float(sd[ks[0]].reshape(-1)[0])])


def fixture_weights(fx):
    """the fixture's weights, regenerated and checked against its checksum: a generator that draws differently fails here"""
    keys = [str(k) for k in fx["keys"]]
    shapes = {k: tuple(int(v) for v in s if v) for k, s in zip(keys, fx["shapes"])}
    sd = weights(int(fx["seed"]), shapes)
    assert np.allclose(wsum(sd), fx["wsum"], rtol=1e-6, atol=1e-6), "regenerated weights differ from the fixture's (torch RNG drift)"
    return sd


def drunet3d_ref64(x, sigma, sd, nb):
    """the reference's forward (drunet.py: m_head .. m_tail with Conv3d / ConvTranspose3d, bias-free) in fp64"""
    sd = {k: v.double() for k, v in sd.items()}
    B = x.shape[0]
    s = torch.as_tensor(sigma, dtype=torch.float64, device=x.device)
    nmap = s.reshape(-1, 1, 1, 1, 1).expand(B, 1, *x.shape[2:]) if s.numel() in (1, B) else s
    t = torch.cat([x.double(), nmap], 1)
    c3 = lambda v, k: F.conv3d(v, sd[k], padding=1)
    rb = lambda v, p: v + c3(F.relu(c3(v, p + ".res.0.weight")), p + ".res.2.weight")

    def blocks(v, name, rng):
        if f"{name}.res.0.weight" in sd:   # nb = 1: the reference unwraps the single body block (m_body.res.*)
            return rb(v, name)
        for i in rng:
            v = rb(v, f"{name}.{i}")
        return v

    x1 = c3(t, "m_head.weight")
    x2 = F.conv3d(blocks(x1, "m_down1", range(nb)), sd[f"m_down1.{nb}.weight"], stride=2)
    x3 = F.conv3d(blocks(x2, "m_down2", range(nb)), sd[f"m_down2.{nb}.weight"], stride=2)
    x4 = F.conv3d(blocks(x3, "m_down3", range(nb)), sd[f"m_down3.{nb}.weight"], stride=2)
    v = blocks(x4, "m_body", range(nb))
    v = blocks(F.conv_transpose3d(v + x4, sd["m_up3.0.weight"], stride=2), "m_up3", range(1, nb + 1))
    v = blocks(F.conv_transpose3d(v + x3, sd["m_up2.0.weight"], stride=2), "m_up2", range(1, nb + 1))
    v = blocks(F.conv_transpose3d(v + x2, sd["m_up1.0.weight"], stride=2), "m_up1", range(1, nb + 1))
    return c3(v + x1, "m_tail.weight")
