"""GPU tests of the fp32 training path: the backward kernels behind `ops._ConvF32Fn` (`dinvk_conv_f32_wgrad`,
`dinvk_relu_bwd`, and the data gradients through the forward entry) at DRUNet / DnCNN layer shapes, and whole-network
gradients of `DRUNet` / `DnCNN` (precision="fp32") and of an unfolded PGD training step, all against a CPU fp64 autograd of
the same fp32 operands.

Yardstick: the reference takes `torch.autograd.grad` of `(out * r).sum()` in fp64; ATen's own CPU fp32 autograd of the
same layer is measured against it too (`e_aten`).  A single layer must satisfy e < 2e-6 and e <= max(4 e_aten, 5e-7).  The
forward kernels, which also compute every data gradient, add their products one after another in fp32 (one chain of 9 Cin
terms per output for a 3x3 layer); such a sum is off by about 0.3 * 2^-24 * sqrt(n) of its size, where ATen's blocked sums
stay near 2.3e-7 (at n = 4608, 512 channels: 1.2e-6 against 2.4e-7).  So the output and the data gradients are held to
max(4 e_aten, 5e-7, 0.5 * 2^-24 * sqrt(n)) under the same 2e-6 cap.  A bias gradient is a sum with cancellation: its error
is measured against the per-channel sums of |g|, the size of its terms.

ReLU masks: fp32 and fp64 disagree on the sign of a pre-activation that lies within rounding of zero, and one such element
moves a gradient by about 1 / sqrt(Cout * B * H * W) of its norm (5e-4 for a 64-channel layer at 4 x 64 x 64; in DnCNN
depth 20 on 2 x 64 x 64, ATen's own fp32 autograd flips one element and lands 2.5e-4 from fp64 in d/dx).  Both answers are
right to fp32 precision, so the fp64 reference applies the ReLU mask of the computation it is compared with (the kernel's
output for the kernel, ATen's for ATen); the number of elements where that mask differs from the fp64 sign is printed.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # fp32 unit roundoff


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


# ---- single layers ---------------------------------------------------------------------------------------------------
def _conv(kind, x, w, bias, xadd, res, relu, mask=None):
    """out = act(conv(x + xadd, w) + bias) + res in plain torch; with `mask` the ReLU keeps exactly the elements where mask"""
    t = x if xadd is None else x + xadd
    if kind == 0:
        y = F.conv2d(t, w, bias, padding=1)
    elif kind == 1:
        y = F.conv2d(t, w, bias, stride=2)
    else:
        y = F.conv_transpose2d(t, w, bias, stride=2)
    if relu:
        y = F.relu(y) if mask is None else y * mask.to(y.dtype)
    return y if res is None else y + res


def _grads(fn, operands, r):
    leaves = {k: v.detach().clone().requires_grad_() for k, v in operands.items()}
    out = fn(leaves)
    g = torch.autograd.grad((out * r).sum(), list(leaves.values()))
    return out.detach(), dict(zip(leaves, g))


def _check_layer(dev, kind, B, Cin, Cout, H, W, *, bias=False, xadd=False, res=False, relu=False, seed=0):
    from deepinv_b200 import ops

    gen = torch.Generator().manual_seed(seed)
    wshape = (Cin, Cout, 2, 2) if kind == 2 else (Cout, Cin, 3, 3) if kind == 0 else (Cout, Cin, 2, 2)
    taps = {0: 9, 1: 4, 2: 1}[kind]
    Ho, Wo = (H, W) if kind == 0 else (H // 2, W // 2) if kind == 1 else (2 * H, 2 * W)
    ops_in = {"x": torch.randn(B, Cin, H, W, generator=gen),
              "w": torch.randn(*wshape, generator=gen) / (taps * Cin) ** 0.5}
    if xadd:
        ops_in["xadd"] = torch.randn(B, Cin, H, W, generator=gen)
    if bias:
        ops_in["bias"] = torch.randn(Cout, generator=gen)
    if res:
        ops_in["res"] = torch.randn(B, Cout, Ho, Wo, generator=gen)
    r = torch.randn(B, Cout, Ho, Wo, generator=gen)

    def plain(mask=None):
        return lambda L: _conv(kind, L["x"], L["w"], L.get("bias"), L.get("xadd"), L.get("res"), relu, mask)

    k_out, k_g = _grads(lambda L: ops.conv_f32_ag(L["x"], L["w"], kind=kind, bias=L.get("bias"), xadd=L.get("xadd"),
                                                  res=L.get("res"), relu=relu),
                        {k: v.to(dev) for k, v in ops_in.items()}, r.to(dev))
    k_out, k_g = k_out.cpu(), {k: v.cpu() for k, v in k_g.items()}
    a_out, a_g = _grads(plain(), ops_in, r)
    o64 = {k: v.double() for k, v in ops_in.items()}
    ref_out, ref_k = _grads(plain(k_out > 0 if relu else None), o64, r.double())
    ref_a = _grads(plain(a_out > 0), o64, r.double())[1] if relu else ref_k
    if relu:
        ref_out = F.relu(ref_out)  # (the masked reference differs from it only where the masks flip: |pre| ~ 1e-7)
    flips = (int(((k_out > 0) != (ref_out > 0)).sum()), int(((a_out > 0) != (ref_out > 0)).sum())) if relu else (0, 0)

    # terms per output of the forward kernel's fp32 chain, and of the data gradient's (the forward kernel of the adjoint)
    n_fwd = {0: 9 * Cin, 1: 4 * Cin, 2: Cin}[kind]
    n_dx = {0: 9 * Cout, 1: Cout, 2: 4 * Cout}[kind]
    seq = {"out": n_fwd, "x": n_dx, "xadd": n_dx}
    errs = {"out": (rel_err(k_out, ref_out), rel_err(a_out, ref_out))}
    for name in k_g:
        if name == "bias":  # against the size of the summed terms: per-channel sums of |g| (g = r behind the ReLU mask)
            def ebias(got, want, mask):
                gabs = (r.double().abs() * (mask if relu else 1.0)).sum(dim=(0, 2, 3))
                return float((got.double() - want).norm() / gabs.norm())
            errs[name] = (ebias(k_g[name], ref_k[name], k_out > 0), ebias(a_g[name], ref_a[name], a_out > 0))
        else:
            errs[name] = (rel_err(k_g[name], ref_k[name]), rel_err(a_g[name], ref_a[name]))
    opts = "".join(f" {o}" for o, on in (("bias", bias), ("xadd", xadd), ("res", res), ("relu", relu)) if on)
    print(f"\nkind {kind} B,Cin,Cout,H,W = {B},{Cin},{Cout},{H},{W}{opts}  ReLU flips vs fp64 (kernel, ATen) {flips}")
    for name, (e_k, e_a) in errs.items():
        floor = 0.5 * U * seq[name] ** 0.5 if name in seq else 0.0
        print(f"  {name:5s} kernel {e_k:.2e}  ATen fp32 {e_a:.2e}")
        assert e_k < 2e-6 and e_k <= max(4 * e_a, 5e-7, floor), (name, e_k, e_a, floor)
    return k_g


LAYERS_3X3 = {  # (B, Cin, Cout, H, W), options
    "drunet_head": ((4, 3, 64, 64, 64), {}),
    "resblock_conv1": ((4, 64, 64, 64, 64), dict(relu=True)),
    "resblock_conv2": ((4, 64, 64, 64, 64), dict(res=True)),
    "level1_relu": ((2, 128, 128, 32, 32), dict(relu=True)),
    "level2_res": ((2, 256, 256, 32, 32), dict(res=True)),
    "level3_relu": ((2, 512, 512, 32, 32), dict(relu=True)),
    "level3_res": ((2, 512, 512, 32, 32), dict(res=True)),
    "drunet_tail": ((4, 64, 2, 64, 64), dict(xadd=True)),
    "dncnn_first": ((4, 1, 64, 40, 56), dict(bias=True, relu=True)),
    "dncnn_middle": ((4, 64, 64, 40, 56), dict(bias=True, relu=True)),  # 8 input-channel chunks: bias from chunk 0 only
    "dncnn_last": ((4, 64, 1, 40, 56), dict(bias=True, res=True)),
    "ragged": ((3, 13, 45, 37, 71), dict(bias=True, xadd=True, relu=True)),  # H % 8, W % 32, Cin % 8, Cout % 32 != 0
    "many_bands": ((8, 64, 64, 128, 128), dict(relu=True)),  # 8 x 16 bands: 128 atomics per weight
    "long_bands": ((1, 8, 32, 9, 1030), dict(bias=True, xadd=True, res=True)),  # 33 tiles per band
}


@pytest.mark.parametrize("case", list(LAYERS_3X3))
def test_conv3x3_layer_gradients_vs_fp64(case, dev):
    shape, opts = LAYERS_3X3[case]
    _check_layer(dev, 0, *shape, **opts)


LAYERS_2X2 = {  # kind, (B, Cin, Cout, H, W) of the layer's input
    "m_down1": (1, (4, 64, 128, 128, 128)),  # M = 16384: 4 chunks of 4096 rows
    "m_up1": (2, (4, 128, 64, 64, 64)),  # M = 16384
    "m_down3": (1, (2, 256, 512, 32, 32)),  # K = 1024
    "m_up3": (2, (2, 512, 256, 16, 16)),  # N = 1024
    "ragged_chunk": (1, (1, 16, 32, 130, 132)),  # M = 4290: a last chunk of 194 rows
}


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("case", list(LAYERS_2X2))
def test_conv2x2_layer_gradients_vs_fp64(case, bias, dev):
    kind, shape = LAYERS_2X2[case]
    _check_layer(dev, kind, *shape, bias=bias, xadd=kind == 2)


# ---- ReLU backward and repeatability ---------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(4, 64, 64, 64), (3, 5, 211, 197)])
def test_relu_bwd_is_threshold_backward_bitwise(shape, dev):
    """n = 1,048,576 and 623,445 (> 148 * 16 blocks of 256: the grid-stride loop takes a second pass, the last one ragged);
    exact zeros of both signs, subnormals, infinities and NaN in `out`, signed zeros and NaN in `g`"""
    from deepinv_b200 import ops

    gen = torch.Generator().manual_seed(11)
    out = torch.randn(shape, generator=gen).relu()  # half exact zeros, as a ReLU output has
    g = torch.randn(shape, generator=gen)
    flat, gf = out.view(-1), g.view(-1)
    flat[1::7] = -0.0
    flat[2::11] = 1e-40
    flat[3::13] = -1e-40
    flat[4::17] = float("inf")
    flat[5::19] = float("-inf")
    flat[6::23] = float("nan")
    gf[7::29] = -0.0
    gf[8::31] = float("nan")
    got = ops.relu_bwd(g.to(dev), out.to(dev)).cpu()
    want = torch.where(out > 0, g, torch.zeros(()))
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("kind,shape", [(0, (8, 64, 64, 128, 128)), (1, (4, 64, 128, 128, 128)), (2, (4, 128, 64, 64, 64))])
def test_wgrad_repeatable(kind, shape, dev):
    """the fp32 atomics make the weight gradient's summation order vary from run to run: two runs agree to 1e-6"""
    from deepinv_b200 import ops

    B, Cin, Cout, H, W = shape
    gen = torch.Generator().manual_seed(4)
    Ho, Wo = (H, W) if kind == 0 else (H // 2, W // 2) if kind == 1 else (2 * H, 2 * W)
    wshape = (Cin, Cout, 2, 2) if kind == 2 else (Cout, Cin, 3, 3) if kind == 0 else (Cout, Cin, 2, 2)
    x = torch.randn(B, Cin, H, W, generator=gen).to(dev)
    g = torch.randn(B, Cout, Ho, Wo, generator=gen).to(dev)
    dw1, db1 = ops.conv_f32_wgrad(x, None, g, wshape, kind=kind, want_bias=True)
    dw2, db2 = ops.conv_f32_wgrad(x, None, g, wshape, kind=kind, want_bias=True)
    e_w, e_b = rel_err(dw1, dw2), rel_err(db1, db2)
    print(f"\nkind {kind} {shape}: run-to-run dw {e_w:.1e}, db {e_b:.1e}")
    assert e_w < 1e-6 and e_b < 1e-6


# ---- whole networks --------------------------------------------------------------------------------------------------
class _ReplayReLU:
    """records the outputs of the package's ReLU convolutions (`ops.conv_f32_ag(..., relu=True)`) and gives the oracle a
    `F` whose `relu` keeps exactly the elements the kernels kept, call by call in the same order"""

    def __init__(self, monkeypatch):
        from deepinv_b200 import ops
        from oracle import ref_ops as R

        self.outs, self.used, self.flips = [], 0, 0
        conv = ops.conv_f32_ag

        def recording(*a, relu=False, **kw):
            out = conv(*a, relu=relu, **kw)
            if relu:
                self.outs.append(out.detach())
            return out

        replay = self

        class _F:
            def __getattr__(self, name):
                return getattr(F, name)

            @staticmethod
            def relu(t):
                keep = replay.outs[replay.used].cpu() > 0
                replay.used += 1
                assert keep.shape == t.shape
                replay.flips += int((keep != (t.detach() > 0)).sum())
                return t * keep.to(t.dtype)

        monkeypatch.setattr(ops, "conv_f32_ag", recording)
        monkeypatch.setattr(R, "F", _F())

    def done(self):
        assert self.used == len(self.outs) > 0, (self.used, len(self.outs))


def _net_params_check(named, ref, tol, what):
    errs = {k: rel_err(p.grad, ref[k].grad) for k, p in named}
    assert len(errs) == len(ref)
    worst = max(errs, key=errs.get)
    print(f"  {what}: {len(errs)} parameter gradients, worst {worst} {errs[worst]:.2e}")
    assert errs[worst] < tol, (worst, errs[worst])


@pytest.mark.parametrize("shape,per_sample_sigma", [((2, 2, 64, 64), True), ((1, 2, 60, 44), False)])
def test_drunet_train_gradients_vs_fp64(shape, per_sample_sigma, dev, monkeypatch):
    """the reference width nc = (64, 128, 256, 512), nb = 2, in train() mode; 60 x 44 goes through the replicate padding"""
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DRUNet(in_channels=2, out_channels=2, nb=2, pretrained=None).train()
    sd64 = {k: v.detach().double().requires_grad_() for k, v in m.state_dict().items()}
    m.to(dev)
    x, r = torch.randn(shape), torch.randn(shape)
    sigma = torch.tensor([0.05, 0.2][: shape[0]]) if per_sample_sigma else 0.1
    replay = _ReplayReLU(monkeypatch)
    xk = x.to(dev).requires_grad_()
    sk = sigma.to(dev).requires_grad_() if per_sample_sigma else sigma
    out = m(xk, sk)
    (out * r.to(dev)).sum().backward()
    x64 = x.detach().double().requires_grad_()
    s64 = sigma.detach().double().requires_grad_() if per_sample_sigma else sigma
    o64 = R.drunet_forward(x64, s64, sd64, nb=2)
    (o64 * r.double()).sum().backward()
    replay.done()
    e_out, e_dx = rel_err(out, o64), rel_err(xk.grad, x64.grad)
    print(f"\nDRUNet {shape}: out {e_out:.2e}, d/dx {e_dx:.2e}, ReLU flips vs fp64 {replay.flips}")
    assert e_out < 1e-5 and e_dx < 1e-5
    if per_sample_sigma:
        e_s = rel_err(sk.grad, s64.grad)
        print(f"  d/dsigma {e_s:.2e}")
        assert e_s < 2e-5
    _net_params_check(m.named_parameters(), sd64, 2e-5, "DRUNet")


def test_dncnn_train_gradients_vs_fp64(dev, monkeypatch):
    import deepinv_b200 as dinv
    from oracle import ref_ops as R

    torch.manual_seed(0)
    m = dinv.models.DnCNN(in_channels=1, out_channels=1, depth=20, nf=64, pretrained=None).train()
    sd64 = {k: v.detach().double().requires_grad_() for k, v in m.state_dict().items()}
    m.to(dev)
    x, r = torch.randn(2, 1, 64, 64), torch.randn(2, 1, 64, 64)
    replay = _ReplayReLU(monkeypatch)
    xk = x.to(dev).requires_grad_()
    out = m(xk)
    (out * r.to(dev)).sum().backward()
    x64 = x.detach().double().requires_grad_()
    o64 = R.dncnn_forward(x64, sd64, depth=20)
    (o64 * r.double()).sum().backward()
    replay.done()
    e_out, e_dx = rel_err(out, o64), rel_err(xk.grad, x64.grad)
    print(f"\nDnCNN depth 20: out {e_out:.2e}, d/dx {e_dx:.2e}, ReLU flips vs fp64 {replay.flips}")
    assert e_out < 1e-5 and e_dx < 1e-5
    _net_params_check(m.named_parameters(), sd64, 2e-5, "DnCNN")


def test_unfolded_pgd_step_vs_fp64(dev, monkeypatch):
    """one training step of unfolded PGD (MRI 64 x 64, B = 2, 2 iterations, trainable stepsize and g_param, full-width
    DRUNet with nb = 1): loss and every gradient against the same loop on the oracle in fp64"""
    import deepinv_b200 as dinv
    from deepinv_b200.optim import L2, PnP
    from deepinv_b200.unfolded import unfolded_builder
    from oracle import ref_ops as R

    torch.manual_seed(0)
    B, H, W = 2, 64, 64
    x = torch.randn(B, 2, H, W)
    cols = (torch.rand(B, 1, 1, W) > 0.7).float()
    cols[..., W // 2 - 3: W // 2 + 3] = 1
    mask = cols.expand(B, 2, H, W).contiguous()
    y = R.mri_A(x, mask)
    den = dinv.models.DRUNet(in_channels=2, out_channels=2, nb=1, pretrained=None).train()
    sd64 = {k: v.detach().double().requires_grad_() for k, v in den.state_dict().items()}
    model = unfolded_builder("PGD", params_algo={"stepsize": [1.0, 0.8], "g_param": [0.05, 0.03], "lambda": 1.0},
                             trainable_params=["stepsize", "g_param"], data_fidelity=L2(), prior=PnP(den), max_iter=2).to(dev)
    algo = {k: list(model.params_algo[k]) for k in ("stepsize", "g_param")}
    algo64 = {k: [p.detach().cpu().double().requires_grad_() for p in v] for k, v in algo.items()}
    replay = _ReplayReLU(monkeypatch)
    phys = dinv.physics.MRI(mask=mask.to(dev), img_size=(2, H, W), device=dev)
    loss = ((model(y.to(dev), phys) - x.to(dev)) ** 2).mean()
    loss.backward()

    y64, m64, x64 = y.double(), mask.double(), x.double()
    aty = R.mri_At(y64, m64)
    xk = aty
    for k in range(2):
        z = xk - algo64["stepsize"][k] * (R.mri_At(R.mri_A(xk, m64), m64) - aty)
        xk = R.drunet_forward(z, algo64["g_param"][k].expand(B), sd64, nb=1)
    loss64 = ((xk - x64) ** 2).mean()
    loss64.backward()
    replay.done()
    e_loss = abs(float(loss.detach()) - float(loss64.detach())) / float(loss64.detach())
    print(f"\nunfolded PGD: loss {e_loss:.2e}, ReLU flips vs fp64 {replay.flips}")
    assert e_loss < 1e-5
    for k in algo:
        got = torch.stack([p.grad.detach().cpu() for p in algo[k]])
        want = torch.stack([p.grad for p in algo64[k]])
        print(f"  d/{k} {rel_err(got, want):.2e}  ({got.tolist()} vs {want.tolist()})")
        assert rel_err(got, want) < 2e-5, k
    _net_params_check(den.named_parameters(), sd64, 2e-5, "DRUNet in the loop")
