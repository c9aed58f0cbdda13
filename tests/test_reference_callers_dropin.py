"""The drop-in classes against what the REFERENCE's own callers compute (SURVEY §8(b) "Callers"): deepinv v0.4.1's optimisers,
data-fidelity terms, least-squares solvers and DDRM sampler were run on the same inputs and their results are stored in
tests/golden/callers_dropin.npz (tests/golden/make_golden.py, callers_fixture); here the drop-in optimisers, sampler and solvers run
on the drop-in operators and denoiser and must reproduce them.  The kernels are the host-emulated SIMT kernels (tests/emul),
injected like in tests/test_host_logic_emul.py."""
import pytest
import torch

import parity_cases as P
from conftest import load_golden, rel_err

DEV = torch.device("cpu")


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


def test_reference_pgd_and_hqs_drive_dropin_mri_and_denoiser():
    """PGD / L2 / PnP over deepinv_b200 MRI.A, A_adjoint, A_adjoint_A, prox_l2 and DRUNet == the reference's PGD on its own MRI and
    DRUNet (same weights); HQS with a closed-form toy denoiser likewise.  Two PGD iterations with the real denoiser keep the
    emulated run short."""
    import deepinv_b200 as dinv

    g = load_golden("optim_mri_tiny")
    want = load_golden("callers_dropin")
    den = P.load_model(dinv.models.DRUNet, g, DEV, in_channels=2, out_channels=2, nc=(8, 16, 32, 64), nb=2)
    phys = dinv.physics.MRI(mask=g["mask"], img_size=(2, 32, 32), device=DEV)
    toy = lambda v, s: v * (1.0 - float(s))
    pgd = dinv.optim.PGD(data_fidelity=dinv.optim.L2(), prior=dinv.optim.PnP(den), stepsize=1.0, sigma_denoiser=0.05, max_iter=2,
                         early_stop=False)
    hqs = dinv.optim.HQS(data_fidelity=dinv.optim.L2(), prior=dinv.optim.PnP(toy), stepsize=0.8, sigma_denoiser=0.05, max_iter=3,
                         early_stop=False)
    with torch.no_grad():
        assert rel_err(pgd(g["y"], phys), want["pgd"]) < 1e-5
        assert rel_err(hqs(g["y"], phys), want["hqs"]) < 1e-5


def test_reference_least_squares_solver_drives_dropin_blur():
    """conjugate gradient on the normal equations through deepinv_b200 Blur.A, A_adjoint, A_adjoint_A == the reference's prox_l2"""
    import deepinv_b200 as dinv

    g = load_golden("blur_gauss_circular_prox")
    phys = dinv.physics.Blur(filter=g["filt"], padding="circular", device=DEV)
    out = dinv.optim.least_squares(phys, g["y"], z=g["z"], init=g["z"], gamma=float(g["gamma"]), solver="CG", max_iter=50, tol=1e-4)
    assert rel_err(out, g["prox"]) < 1e-4


def test_reference_ddrm_drives_dropin_mri():
    """DDRM (sampling/diffusion.py:149-224) over deepinv_b200 MRI.U_adjoint / V / V_adjoint / mask == the reference's DDRM on its
    own MRI: recorded noise draws, closed-form toy denoiser"""
    import deepinv_b200 as dinv

    g = load_golden("ddrm_mri_tiny")
    toy = lambda v, s: v * (1.0 / (1.0 + float(s)))
    sig = float(g["sigma_noise"])
    phys = dinv.physics.MRI(mask=g["mask"], img_size=(2, 32, 32), device=DEV, noise_model=dinv.physics.GaussianNoise(sigma=sig))
    it = iter(list(g["noises"]))
    orig = torch.randn_like
    torch.randn_like = lambda t, **kw: next(it).to(t)
    try:
        out = dinv.sampling.DDRM(denoiser=toy, sigmas=g["sigmas"].numpy())(g["y"], phys)
    finally:
        torch.randn_like = orig
    assert rel_err(out, load_golden("callers_dropin")["ddrm"]) < 1e-5


@pytest.mark.parametrize("solver", ["CG", "BiCGStab"])
def test_least_squares_solvers_match_the_reference_solvers(solver):
    """deepinv_b200.optim.least_squares (CG / BiCGStab on the kernels) == the reference's least_squares with the same solver on the
    same operator (the reference's own Blur): same iterates, same stopping rule"""
    import deepinv_b200 as dinv

    g = load_golden("blur_gauss_circular_prox")
    ref = load_golden("callers_dropin")
    phys = dinv.physics.Blur(filter=g["filt"], padding="circular", device=DEV)
    gam = float(g["gamma"])
    want = ref[f"ls_{solver}"]
    got = dinv.optim.least_squares(phys, g["y"], z=g["z"], init=g["z"], gamma=gam, solver=solver, max_iter=25, tol=1e-5)
    # CG: regularised normal equations, well conditioned.  BiCGStab on this square operator: the UNregularised deblurring system
    # A x = y (see below) — 40 iterations of it amplify the round-off differences of the inner products to a few 1e-4
    assert rel_err(got, want) < (2e-5 if solver == "CG" else 2e-3)
    if solver == "CG":
        assert rel_err(got, g["prox"]) < 1e-3  # the fixture was produced with tol = 1e-4 (LinearPhysics default)
    else:  # complete system: the reference gives BiCGStab A x = y itself (gamma, z unused) — so does the drop-in
        assert rel_err(phys.A(got), g["y"]) < 1e-3
        valid = dinv.physics.Blur(filter=g["filt"], padding="valid", device=DEV)   # rectangular: normal equations with gamma
        yv = valid.A(g["z"])
        assert rel_err(yv, ref["yv"]) < 1e-6
        want_v = ref["ls_BiCGStab_valid"]
        got_v = dinv.optim.least_squares(valid, yv, z=g["z"], init=g["z"], gamma=gam, solver=solver, max_iter=25, tol=1e-5)
        assert rel_err(got_v, want_v) < 2e-5


def test_lsqr_matches_the_reference_lsqr_on_a_rectangular_operator():
    """deepinv_b200.optim.lsqr (Golub-Kahan on the kernels) vs the reference's lsqr (optim/linear/lsqr.py) on the drop-in valid-padding
    Blur (rectangular): damped problem with a warm start, and the plain pseudo-inverse"""
    import deepinv_b200 as dinv

    g = load_golden("blur_gauss_circular_prox")
    ref = load_golden("callers_dropin")
    phys = dinv.physics.Blur(filter=g["filt"], padding="valid", device=DEV)
    y = ref["y_lsqr"]   # the reference's valid-padding blur of z + seeded noise
    assert rel_err(y - phys.A(g["z"]), ref["y_lsqr"] - ref["yv"]) < 1e-4
    for gam, batched in ((2.0, False), (torch.tensor([0.5, 3.0]), True)):
        want = ref["lsqr_batched" if batched else "lsqr_scalar"]
        got = dinv.optim.least_squares(phys, y, z=g["x"], init=g["x"], gamma=gam, solver="lsqr", max_iter=30, tol=1e-6)
        assert rel_err(got, want) < 1e-4, batched
    cg = dinv.optim.least_squares(phys, y, z=g["x"], init=g["x"], gamma=2.0, solver="CG", max_iter=60, tol=1e-6)
    assert rel_err(dinv.optim.least_squares(phys, y, z=g["x"], gamma=2.0, solver="lsqr", max_iter=60, tol=1e-7), cg) < 1e-3


def test_minres_matches_the_reference_minres():
    """deepinv_b200.optim.minres vs the reference's minres (optim/linear/minres.py): the symmetric system (A^T A + I/gamma) x = b of a
    rectangular operator through least_squares, and a symmetric complete operator handed over as A x = y"""
    import deepinv_b200 as dinv

    g = load_golden("blur_gauss_circular_prox")
    ref = load_golden("callers_dropin")
    valid = dinv.physics.Blur(filter=g["filt"], padding="valid", device=DEV)
    y = valid.A(g["z"])
    want = ref["minres_valid"]
    got = dinv.optim.least_squares(valid, y, z=g["x"], init=g["x"], gamma=2.0, solver="minres", max_iter=30, tol=1e-6)
    assert rel_err(got, want) < 1e-4
    circ = dinv.physics.Blur(filter=g["filt"], padding="circular", device=DEV)  # symmetric filter: A = A^T, complete system
    want = ref["minres_circ"]
    got = dinv.optim.least_squares(circ, g["y"], z=g["z"], init=g["z"], gamma=2.0, solver="minres", max_iter=15, tol=1e-6)
    assert rel_err(got, want) < 2e-3  # unregularised deblurring: see the BiCGStab case above
