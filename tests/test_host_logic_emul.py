"""Host-side logic without a GPU: the package's own Python code (physics classes, optimisers, denoisers,
sampler) driving the EMULATED kernels (tests/emul) on CPU tensors, checked against the reference's golden
vectors.  The emulated backend is injected by monkeypatching three private hooks of deepinv_b200.ops inside
this test session only; the package itself has no CPU switch (see tests/test_abi.py::test_no_cpu_fallback)."""
import pytest
import torch

import parity_cases as P
from conftest import golden_names


@pytest.fixture(autouse=True)
def emul_backend(monkeypatch):
    from emul_util import emul_lib

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


DEV = torch.device("cpu")


@pytest.mark.parametrize("name", golden_names("mri_"))
def test_mri(name):
    P.case_mri(name, DEV)


@pytest.mark.parametrize("name", golden_names("dynmri_") + golden_names("seqmri_"))
def test_dynamic_mri(name):
    P.case_dynamic_mri(name, DEV)


@pytest.mark.parametrize("name", golden_names("fan_"))
def test_fanbeam(name):
    P.case_fanbeam(name, DEV)


@pytest.mark.parametrize("name", golden_names("down_"))
def test_downsampling(name):
    P.case_downsampling(name, DEV)


def test_combine():
    P.case_combine(DEV)


def test_mri_3d():
    P.case_mri_3d(DEV)


def test_anderson():
    P.case_anderson(DEV, full=False)


def test_filters():
    P.case_filters(DEV)


@pytest.mark.parametrize("name", golden_names("mcmri_"))
def test_multicoil(name):
    P.case_multicoil(name, DEV)


@pytest.mark.parametrize("name", ["tomo_16_a8", "tomo_24_a10_circle"])
def test_tomography(name):
    P.case_tomography(name, DEV)


def test_tomography_normalised():
    P.case_tomography_normalised(DEV)


@pytest.mark.parametrize("name", ["blur_3x3_valid", "blur_4x4_circular", "blur_5x3_replicate", "blur_6x5_reflect",
                                  "blur_4x4_constant", "blur_5x5_perbc_reflect"])
def test_blur(name):
    P.case_blur(name, DEV)


def test_blur_cg():
    P.case_blur_cg(DEV)


@pytest.mark.parametrize("name", ["blurfft_18x20", "blurfft_15x16_odd", "blurfft_persample", "blurfft_persample_c"])
def test_blurfft(name):
    P.case_blurfft(name, DEV)


def test_drunet():
    P.case_drunet(DEV)


def test_dncnn():
    P.case_dncnn(DEV)


def test_pnp_mri():
    P.case_pnp_mri(DEV, full=False)


def test_drs_gd_dpir():
    P.case_drs_gd_dpir(DEV, full=False)


def test_train_deq_explicit():
    P.case_train_deq_explicit(DEV)


def test_pnp_blur_admm():
    P.case_pnp_blur_admm(DEV)


def test_ddrm_inpainting_and_denoising():
    P.case_ddrm_inpainting(DEV)


def test_pdcp():
    P.case_pdcp(DEV)


def test_diffpir():
    P.case_diffpir(DEV)


def test_optim_step_algebra_toy_denoiser():
    P.case_optim_toy(DEV)


def test_dpir_schedule_toy_denoiser():
    """DPIR's per-iteration (sigma, stepsize) schedule and HQS step algebra with a closed-form 'denoiser' (the real
    DRUNet run is the GPU case): package loop on emulated kernels == oracle loop"""
    from conftest import load_golden, rel_err
    from oracle import ref_ops as R

    import deepinv_b200 as dinv
    from deepinv_b200.optim import DPIR, get_DPIR_params

    g = load_golden("optim2_mri_tiny")
    m, y = g["mask"], g["y"]
    den = lambda v, s: v * (1.0 - float(s))
    phys = dinv.physics.MRI(mask=m, img_size=(2, 32, 32), device=DEV)
    model = DPIR(sigma=0.05, denoiser=den, device=DEV)
    sig, step, n = get_DPIR_params(0.05)
    rs, rt, rn = R.dpir_params(0.05)
    assert n == rn == 8 and torch.equal(sig, rs) and torch.equal(step, rt)
    # DPIR's first stepsizes are large (gamma = 64 at iteration 0): (A^T y + z/gamma) / (s^2 + 1/gamma) then loses ~3e-6 in
    # fp32 per prox for ANY implementation, the reference's included.  So the comparison is against the fp64 evaluation of
    # the same recipe, and the package must be as close to it as the fp32 reference path is.
    y64, m64 = y.double(), m.double()
    truth = R.dpir(y64, lambda v, gam: R.mri_prox_l2(v, y64, m64, float(gam)), lambda v: R.mri_At(v, m64), den, 0.05)
    ref32 = R.dpir(y, lambda v, gam: R.mri_prox_l2(v, y, m, gam), lambda v: R.mri_At(v, m), den, 0.05)
    e_ref, e_pkg = rel_err(ref32, truth), rel_err(model(y, phys), truth)
    assert e_pkg < max(2 * e_ref, 1e-5) and e_pkg < 5e-5, (e_pkg, e_ref)


# ---- SURVEY §8(f) item 2: training closure (backward kernels of the fp32 denoiser path) ---------------------------
@pytest.mark.parametrize("kind,cin,cout,h,w", [(0, 5, 7, 11, 37), (0, 16, 40, 16, 64), (1, 6, 10, 8, 12), (2, 10, 6, 5, 7),
                                               (1, 3, 5, 96, 98), (2, 5, 3, 48, 50)])
def test_conv_backward_kernels(kind, cin, cout, h, w):
    """data / weight / bias / residual / skip-input gradients of `ops.conv_f32_ag` == torch autograd of the same op.  The last
    two shapes have M = 4704 and 4800 pixel rows: the 2x2 weight gradient then runs two 4096-row chunks, the second ragged."""
    import torch.nn.functional as F
    from conftest import rel_err

    from deepinv_b200 import ops

    torch.manual_seed(kind * 7 + cin)
    B = 2
    x = torch.randn(B, cin, h, w, requires_grad=True)
    xadd = torch.randn(B, cin, h, w, requires_grad=True)
    wshape = (cin, cout, 2, 2) if kind == 2 else (cout, cin, 3, 3) if kind == 0 else (cout, cin, 2, 2)
    wt = (torch.randn(wshape) / 4).requires_grad_()
    bias = torch.randn(cout, requires_grad=True)
    for relu, use_res in ((True, False), (False, True)):
        conv = {0: lambda t: F.conv2d(t, wt, bias, padding=1), 1: lambda t: F.conv2d(t, wt, bias, stride=2),
                2: lambda t: F.conv_transpose2d(t, wt, bias, stride=2)}[kind]
        ref = conv(x + xadd)
        res = torch.randn_like(ref).requires_grad_() if use_res else None
        ref = torch.relu(ref) if relu else ref
        ref = ref + res if use_res else ref
        r = torch.randn_like(ref)
        leaves = [x, xadd, wt, bias] + ([res] if use_res else [])
        want = torch.autograd.grad((ref * r).sum(), leaves)
        out = ops.conv_f32_ag(x, wt, kind=kind, bias=bias, xadd=xadd, res=res, relu=relu)
        assert rel_err(out, ref) < 1e-5
        got = torch.autograd.grad((out * r).sum(), leaves)
        for a, b in zip(got, want):
            assert a.shape == b.shape and rel_err(a, b) < 1e-5


def test_drunet_gradients():
    """d loss / d (input, every weight) of the tiny DRUNet through the library's backward == autograd of the oracle"""
    from conftest import load_golden, rel_err
    from oracle import ref_ops as R

    import deepinv_b200 as dinv

    g = load_golden("drunet_tiny")
    den = P.load_model(dinv.models.DRUNet, g, DEV, in_channels=2, out_channels=2, nc=(8, 16, 32, 64), nb=2)
    x = g["x"][:1, :, :, :32].clone().requires_grad_()
    r = torch.randn(1, 2, 32, 32)
    (den(x, 0.05) * r).sum().backward()
    sd = {k: v.clone().requires_grad_() for k, v in g["sd"].items()}
    x2 = x.detach().clone().requires_grad_()
    (R.drunet_forward(x2, 0.05, sd, nb=2) * r).sum().backward()
    assert rel_err(x.grad, x2.grad) < 1e-5
    for k, p in den.named_parameters():
        assert rel_err(p.grad, sd[k].grad) < 2e-5, k


@pytest.mark.parametrize("batched_gamma", [False, True])
def test_least_squares_implicit_backward(batched_gamma):
    """prox_l2 of a non-decomposable operator (circular Blur, CG on the kernels): value and the implicit-differentiation
    gradients w.r.t. y, z, gamma == autograd through a dense fp64 solve of the same normal equations"""
    from conftest import rel_err
    from oracle import ref_ops as R

    import deepinv_b200 as dinv

    torch.manual_seed(3)
    B, H, W = 2, 8, 10
    filt = torch.rand(1, 1, 3, 3)
    filt = filt / filt.sum()
    phys = dinv.physics.Blur(filter=filt, padding="circular", device=DEV)
    phys.max_iter, phys.tol = 25, 1e-5
    y = torch.randn(B, 1, H, W, requires_grad=True)
    z = torch.randn(B, 1, H, W, requires_grad=True)
    gamma = (torch.tensor([0.7, 2.5]) if batched_gamma else torch.tensor(1.3)).requires_grad_()
    r = torch.randn(B, 1, H, W)
    out = phys.prox_l2(z, y, gamma)
    gy, gz, gg = torch.autograd.grad((out * r).sum(), [y, z, gamma])
    # dense reference
    n = H * W
    eye = torch.eye(n, dtype=torch.float64).reshape(n, 1, H, W)
    A = R.blur_A(eye.float(), filt, "circular").double().reshape(n, n).T  # columns = A e_i
    y64, z64, g64 = (t.detach().double().requires_grad_() for t in (y, z, gamma))
    gb = g64.reshape(-1, 1) if batched_gamma else g64
    rhs = y64.reshape(B, n) @ A + z64.reshape(B, n) / gb
    hs = []
    for b in range(B):
        gcur = g64[b] if batched_gamma else g64
        hs.append(torch.linalg.solve(A.T @ A + torch.eye(n, dtype=torch.float64) / gcur, rhs[b]))
    h = torch.stack(hs).reshape(B, 1, H, W)
    wy, wz, wg = torch.autograd.grad((h * r.double()).sum(), [y64, z64, g64])
    assert rel_err(out, h) < 1e-5
    assert rel_err(gy, wy) < 2e-4 and rel_err(gz, wz) < 2e-4 and rel_err(gg, wg) < 2e-4


def test_memoised_adjoint_is_not_served_for_a_new_tensor_at_the_same_address():
    """regression: prox_l2 memoises A^T y per measurement tensor; a freed y whose address is handed to the next y (same
    shape, version 0) must not hit the stale entry — the cache key holds the tensor itself, not its pointer"""
    from conftest import load_golden, rel_err
    from oracle import ref_ops as R

    import deepinv_b200 as dinv

    g = load_golden("optim2_mri_tiny")
    m = g["mask"]
    phys = dinv.physics.MRI(mask=m, img_size=(2, 32, 32), device=DEV)
    z = torch.randn(2, 2, 32, 32)
    seen = set()
    for k in range(6):
        y = R.mri_A(torch.randn(2, 2, 32, 32), m).clone()  # freed at the end of the iteration: the allocator reuses the block
        seen.add(y.data_ptr())
        assert rel_err(phys.prox_l2(z, y, 0.7), R.mri_prox_l2(z, y, m, 0.7)) < 1e-5
        del y
    y = R.mri_A(torch.randn(2, 2, 32, 32), m)
    a = phys.prox_l2(z, y, 0.7)
    y.mul_(2.0)  # in-place change of the SAME tensor: version bump -> recomputed
    assert rel_err(phys.prox_l2(z, y, 0.7), R.mri_prox_l2(z, y, m, 0.7)) < 1e-5 and rel_err(a, phys.prox_l2(z, y, 0.7)) > 1e-2


def test_lsqr_degenerate_sample_in_batch():
    """a zero measurement inside a batch (padded sample) must not poison that sample with NaN (the reference returns early for it,
    optim/linear/lsqr.py:150-160) and must not change the other samples"""
    import deepinv_b200 as dinv

    torch.manual_seed(0)
    filt = torch.rand(1, 1, 3, 3)
    filt /= filt.sum()
    phys = dinv.physics.Blur(filter=filt, padding="valid", device=DEV)
    x = torch.randn(3, 1, 12, 14)
    y = phys.A(x)
    y[1] = 0
    got = dinv.optim.least_squares(phys, y, solver="lsqr", max_iter=40, tol=1e-7)
    assert torch.isfinite(got).all()
    assert float(got[1].abs().max()) == 0.0
    alone = dinv.optim.least_squares(phys, y[[0, 2]], solver="lsqr", max_iter=40, tol=1e-7)
    # (the stopping rule is evaluated over the batch: same iteration count here because sample 1 is converged from the start)
    assert torch.allclose(got[[0, 2]], alone, rtol=1e-5, atol=1e-6)


def test_workspace_growth_keeps_outgrown_buffers_alive():
    """a CUDA graph captured earlier has the old workspace address baked in: growing must not free it (ops.workspace)"""
    from deepinv_b200 import ops

    ops._ws_cache.clear()
    a = ops.workspace(DEV, 64, "t")
    pa = a.data_ptr()
    b = ops.workspace(DEV, 4096, "t")
    assert b.numel() >= 4096 and any(t.data_ptr() == pa for t in ops._ws_retired)
