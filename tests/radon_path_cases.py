"""One case table for every launch path of the Radon family (csrc/radon.cu) and the ramp filter (csrc/spectral.cu), shared by
the H100 run (tests/test_gpu_radon_paths.py) and the host-emulated twin (tests/test_emul_radon_paths.py).

The host code picks a kernel from the image width, the angle count and the input's alignment: the tiled kernels
(`radon_tiled_kernel<false/true>`, W >= 64, W % 4 == 0, A <= 2048, 16-byte aligned input; the forward stages its tile by TMA
or, under DINVK_NO_TMA_STAGING, by a mapped loop), the per-ray kernels (`radon_fwd_kernel`, `radon_adj_kernel`) otherwise or
under DINVK_NO_TILED_RADON, the IRadon back-projection (`iradon_bp_kernel`), the fan-beam pair (`fanbeam_kernel<false/true>`),
and the ramp filter's exact spatial kernel (N <= 8192) or its FFT form (DINVK_RAMP_FFT: mean subtraction, row pass, box
response).  Each row names the call, the kernel it must reach and the number of launches the host issues.  The launch count
pins the host branch; the kernel census of the GPU file pins the kernel of every row.

Every row is checked against the fp64 restatement (tests/radon_ref64.py), per image:
  * forwards: relative L2 <= 1e-6; exact transposes: <= 5e-6 (the tiled transpose beyond 360 angles: 5e-6 * A / 360, its
    fixed-point unit grows with A); both: max |error| <= 2e-5 * max |ref|;
  * IRadon and fan beam (fp32 geometry of the reference's formulas): relative L2 < 1e-5 against the oracle in fp32, or an
    error against the fp64 restatement of at most 1.15 x the oracle's own fp32 error + 2e-7;
  * ramp filter: exact kernel <= 1e-7, FFT form <= 1e-5;
  * offset inputs agree with the same call on aligned memory to 3e-7;
  * non-finite inputs: every output that a NaN / +Inf / -Inf reaches with an fp64 weight above 1e-6 is non-finite, and every
    output more than 2 pixels (transposes) or 2 detector cells (forwards) from all outputs it reaches is finite and within the
    row's tolerance of the same call with the non-finite values replaced by zeros;
  * Aᵀ(2^k y) == 2^k Aᵀ(y) bit for bit (the tiled transpose's fixed-point scale follows the data).
"""
from __future__ import annotations

import dataclasses
import json
import math
import os
import subprocess
import sys
import zlib
from pathlib import Path
from typing import Optional

import torch

import radon_ref64 as RR

TOL_FWD, TOL_ADJ, TOL_MAX = 1e-6, 5e-6, 2e-5
TOL_RAMP, TOL_RAMP_FFT = 1e-7, 1e-5
TOL_ORACLE = 1e-5
HERE = Path(__file__).resolve().parent

K_TILED_F, K_TILED_A = "radon_tiled_kernel<false>", "radon_tiled_kernel<true>"
K_RAY_F, K_RAY_A, K_IRADON = "radon_fwd_kernel", "radon_adj_kernel", "iradon_bp_kernel"
K_FAN_F, K_FAN_A = "fanbeam_kernel<false>", "fanbeam_kernel<true>"
K_RAMP = "ramp_exact_kernel"

NO_TMA = (("DINVK_NO_TMA_STAGING", "1"),)
NO_TILED = (("DINVK_NO_TILED_RADON", "1"),)

ANGLES_USER = (170.0, -30.0, 200.0, 45.5, 200.0, 10.0, -190.0, 359.0, 91.25, 0.75)
ANGLES_EXACT = (0.0, 45.0, 90.0)
ANGLES_NEAR = (1e-5, -1e-5, 1e-4, 1e-3, -1e-3, 90 - 1e-5, 90 + 1e-5, 90 - 1e-4, 90 + 1e-3, 180 - 1e-5)
WIDE_FAN = {"n_detector_pixels": 301, "detector_spacing": 0.2, "source_radius": 30.0, "detector_radius": 20.0}


@dataclasses.dataclass(frozen=True)
class Row:
    name: str
    call: str             # A | At | At_ir | fbp_ir | fanA | fanAt | ramp | raw_A (forward of an offset view)
    W: int                # image width (ramp rows: the row length N)
    A: object             # angle count, or a tuple of angles in degrees (ramp rows: the number of rows per image)
    kernels: tuple        # the kernels the row must launch (GPU census)
    launches: int
    circle: bool = False
    bc: tuple = (2, 1)    # (B, C)
    env: tuple = ()
    data: str = "randn"   # randn | const | alt | point | nonfinite | bitexact | ramp
    fan: Optional[dict] = None
    error: str = ""       # the call must raise DinvkError with this text
    emul: Optional[tuple] = None   # (W, A) for the host emulation, on the same path
    gpu_only: str = ""    # why the emulation cannot check this row

    @property
    def nang(self):
        return self.A if isinstance(self.A, int) else len(self.A)


def _rows():
    R = []
    # ---- tiled kernels, TMA staging (the forward) / the fixed-point transpose ---------------------------------------------
    tiled = [("64", 64, 30, False, (2, 1), None), ("68 4-pixel last tile", 68, 24, False, (2, 1), None),
             ("124", 124, 20, False, (1, 1), None), ("256", 256, 45, False, (2, 1), (128, 12)),
             ("512 cfg3", 512, 180, False, (1, 1), (132, 6)), ("1024 P1449", 1024, 3, False, (1, 1), (192, 2)),
             ("circle 128", 128, 40, True, (2, 1), None), ("circle 100", 100, 30, True, (1, 1), None),
             ("96 C3", 96, 16, False, (2, 3), None), ("64 A1", 64, 1, False, (2, 1), None),
             ("64 A2048", 64, 2048, False, (1, 1), (64, 300))]
    for tag, W, A, circ, bc, em in tiled:
        R.append(Row(f"tiled {tag} A", "A", W, A, (K_TILED_F,), 1, circ, bc, emul=em))
        R.append(Row(f"tiled {tag} A mapped", "A", W, A, (K_TILED_F,), 1, circ, bc, env=NO_TMA, emul=em))
        R.append(Row(f"tiled {tag} At", "At", W, A, (K_TILED_A,), 1, circ, bc, emul=em))
    # ---- per-ray kernels: W < 64, W % 4 == 2, an odd-width circle, more than 2048 angles, the 48 KB shared-memory line --------
    for tag, W, circ in (("62", 62, False), ("66", 66, False), ("circle 63", 63, True)):
        R += [Row(f"ray {tag} A", "A", W, 20, (K_RAY_F,), 1, circ),
              Row(f"ray {tag} At", "At", W, 20, (K_RAY_A,), 1, circ)]
    smem = "the emulation has no 48 KB shared-memory limit: only the H100 sees whether the launch opts in"
    for A in (2049, 3072, 3073, 4096):  # W = 64 would take the tiled kernels but for the angle count
        big = A > 3072
        R += [Row(f"ray 64 A{A} A", "A", 64, A, (K_RAY_F,), 1, bc=(1, 1), emul=(16, A)),
              Row(f"ray 64 A{A} At", "At", 64, A, (K_RAY_A,), 1, bc=(1, 1), emul=(16, A), gpu_only=smem if big else "")]
    R.append(Row("iradon 64 A4096 At", "At_ir", 64, 4096, (K_IRADON,), 1, bc=(1, 1), emul=(16, 4096)))
    R += [Row("ray 64 A4097 At", "At", 64, 4097, (), 0, bc=(1, 1), error="grid too large"),
          Row("iradon 64 A4097 At", "At_ir", 64, 4097, (), 0, bc=(1, 1), error="grid too large")]
    R.append(Row("ray 128 offset input A", "raw_A", 128, 24, (K_RAY_F, K_TILED_F), 1, emul=(64, 8)))
    for tag, W, A, circ in (("128", 128, 40, False), ("200 circle", 200, 30, True)):
        R += [Row(f"no-tiled {tag} A", "A", W, A, (K_RAY_F,), 1, circ, env=NO_TILED, emul=(64, 10)),
              Row(f"no-tiled {tag} At", "At", W, A, (K_RAY_A,), 1, circ, env=NO_TILED, emul=(64, 10))]
    # ---- angles: user-given (unsorted, negative, above 180, duplicated), exact 0 / 45 / 90, within 1e-5 .. 1e-3 of 0 and 90 ---
    for atag, ang in (("user", ANGLES_USER), ("exact", ANGLES_EXACT), ("near", ANGLES_NEAR)):
        R += [Row(f"angles {atag} tiled 128 A", "A", 128, ang, (K_TILED_F,), 1, emul=(64, ang)),
              Row(f"angles {atag} tiled 128 At", "At", 128, ang, (K_TILED_A,), 1, emul=(64, ang)),
              Row(f"angles {atag} ray 66 A", "A", 66, ang, (K_RAY_F,), 1),
              Row(f"angles {atag} ray 66 At", "At", 66, ang, (K_RAY_A,), 1)]
    # ---- IRadon back-projection (adjoint_via_backprop=False): A_adjoint and FBP --------------------------------------------
    for W, A in ((256, 180), (512, 60)):
        R += [Row(f"iradon {W} At", "At_ir", W, A, (K_IRADON,), 1, bc=(1, 1), emul=(64, 20)),
              Row(f"iradon {W} fbp", "fbp_ir", W, A, (K_RAMP, K_IRADON), 2, bc=(1, 1), emul=(64, 20))]
    # ---- fan beam: default geometry and a wide fan ---------------------------------------------------------------------------
    for W in (128, 256):
        for ftag, fp in (("default", None), ("wide", WIDE_FAN)):
            R += [Row(f"fan {W} {ftag} A", "fanA", W, 24, (K_FAN_F,), 1, fan=fp, emul=(32, 6)),
                  Row(f"fan {W} {ftag} At", "fanAt", W, 24, (K_FAN_A,), 1, fan=fp, emul=(32, 6))]
    # ---- ramp filter, exact kernel: N = 1, 2, 3, 725, 1449 and 8192 (98 KB of shared memory), odd row counts, one row -------
    for N, rows, bc, em in ((1, 5, (1, 1), None), (2, 3, (1, 2), None), (3, 4, (2, 1), None), (725, 180, (1, 1), (725, 20)),
                            (1449, 31, (1, 1), (1449, 7)), (8192, 6, (1, 1), (8192, 2)), (725, 1, (1, 1), None)):
        R.append(Row(f"ramp exact N{N} rows{rows * bc[0] * bc[1]}", "ramp", N, rows, (K_RAMP,), 1, bc=bc, data="ramp", emul=em))
    # ---- the tiled transpose's fixed-point accumulator: its range, its precision, its scale ---------------------------------
    for d in ("const", "alt", "point"):
        R.append(Row(f"fixed-point {d} tiled 128 At", "At", 128, 60, (K_TILED_A,), 1, data=d, emul=(64, 20)))
    R.append(Row("fixed-point 2^k equivariance tiled 64 At", "At", 64, 90, (K_TILED_A,), 1, data="bitexact"))
    # ---- non-finite values: one NaN, one +Inf, one -Inf in image 0 of each forward's input / each transpose's sinogram -------
    nf = [("tiled 128 At", "At", 128, (K_TILED_A,), (), None), ("ray 66 At", "At", 66, (K_RAY_A,), (), None),
          ("iradon 128 At", "At_ir", 128, (K_IRADON,), (), (64, 16)), ("fan 128 At", "fanAt", 128, (K_FAN_A,), (), (32, 8)),
          ("tiled 128 A", "A", 128, (K_TILED_F,), (), None), ("tiled 128 A mapped", "A", 128, (K_TILED_F,), NO_TMA, None),
          ("ray 66 A", "A", 66, (K_RAY_F,), (), None), ("fan 128 A", "fanA", 128, (K_FAN_F,), (), (32, 8))]
    for tag, call, W, k, env, em in nf:
        R.append(Row(f"non-finite {tag}", call, W, 24, k, 1, env=env, data="nonfinite", emul=em or (64 if W == 128 else W, 12)))
    names = [r.name for r in R]
    assert len(names) == len(set(names)), [n for n in names if names.count(n) > 1]
    return R


ROWS = _rows()

# FFT form of the ramp filter: DINVK_RAMP_FFT is read once per process, so these run in one child process (run_fft_rows).
# (N, rows): odd and even row counts; "ws": through ops.ramp_filter (mean-free, with its workspace) or the raw ABI without one
FFT_ROWS = [(N, rows, ws) for N in (725, 1449) for rows in (6, 7) for ws in (True, False)]
# past the exact kernel's N <= 8192 the FFT form takes over; at N = 8193 its padded length does not fit a row tile
N8193 = "dinvk_ramp_filter: padded length 32768 too large"


# ------------------------------------------------------------------------------------------------------------------------------
# inputs, calls, references
# ------------------------------------------------------------------------------------------------------------------------------
def _angles(A):
    if isinstance(A, int):
        return torch.linspace(0, 180, steps=A + 1)[:-1]  # Tomography's default (tomography.py:136-139)
    return torch.tensor(A, dtype=torch.float32)


class Case:
    def __init__(self, row: Row, dev: torch.device, emulated: bool = False):
        self.row, self.dev = row, dev
        W, A = (row.emul if emulated and row.emul else (row.W, row.A))
        self.W, self.A = W, A
        self.ang = _angles(A)
        self.nang = len(self.ang)
        self.g = torch.Generator().manual_seed(zlib.crc32(row.name.encode()))
        B, C = row.bc
        r = row
        if r.call == "ramp":
            u = torch.linspace(-1, 1, W).clamp(-1, 1)
            prof = 30 * (1 - u * u).clamp_min(0).sqrt()
            self.inp = prof + torch.randn(B, C, A, W, generator=self.g)
            return
        self.fan = RR.fan_constants(W, r.circle, r.fan) if r.call.startswith("fan") else None
        self.P = self.fan[2] if self.fan else RR.geometry(W, r.circle)[0]
        fwd = r.call in ("A", "fanA", "raw_A")
        shape = (B, C, W, W) if fwd else (B, C, self.nang, self.P)
        g = self.g
        if r.data in ("randn", "nonfinite", "bitexact"):
            self.inp = torch.randn(shape, generator=g)
        elif r.data == "const":
            self.inp = torch.ones(shape)
        elif r.data == "alt":
            t = torch.arange(self.nang)[:, None] + torch.arange(self.P)[None, :]
            self.inp = (1 - 2 * (t % 2)).float().expand(shape).contiguous()
        elif r.data == "point":
            d = torch.zeros(B, C, W, W, dtype=torch.float64)
            d[..., W // 3, W // 2] = 1.0
            self.inp = (RR.radon_fwd(d, self.ang, r.circle) + 1e-3 * torch.randn(shape, generator=g, dtype=torch.float64)).float()
        self.bad = []
        if r.data == "nonfinite":
            self._place_nonfinite(fwd)

    def _place_nonfinite(self, fwd):
        W = self.W
        if fwd:  # three pixels inside the disc of image 0
            locs = [(W // 2, W // 3), (W // 3 + 1, (2 * W) // 3), ((2 * W) // 3, W // 2 + 3)]
        else:  # three rays of image 0 that cross the image
            P, A = self.P, self.nang
            locs = [(1, P // 2 - 3), (A // 2, P // 2 + 5), (A - 2, P // 3 + 2)]
        for (a, b), v in zip(locs, (float("nan"), float("inf"), float("-inf"))):
            self.inp[0, 0, a, b] = v
            self.bad.append((a, b))

    # ---- the call under test ----------------------------------------------------------------------------------------------
    def _phys(self, **kw):
        import deepinv_b200 as dinv

        r = self.row
        ang = self.A if isinstance(self.A, int) else self.ang
        return dinv.physics.Tomography(angles=ang, img_width=self.W, circle=r.circle, normalize=False, device=self.dev,
                                       fan_beam=r.call.startswith("fan"), fan_parameters=r.fan, **kw)

    def make_call(self, inp=None):
        """the call of the row as a closure (physics objects are built outside it); outputs are angle-major for forwards"""
        from deepinv_b200 import ops

        r = self.row
        x = (self.inp if inp is None else inp).to(self.dev)
        if r.call == "ramp":
            return lambda: ops.ramp_filter(x)
        if r.call == "raw_A":
            flat = torch.zeros(x.numel() + 1, device=self.dev)
            flat[1:] = x.reshape(-1)
            x = flat[1:].view(x.shape)
        phys = self._phys(adjoint_via_backprop=r.call not in ("At_ir", "fbp_ir"))
        phys._trig()
        if r.call in ("A", "fanA", "raw_A"):
            return lambda: phys.A(x).transpose(-2, -1)
        y = x.transpose(-2, -1)  # the (B, C, P, A) view Tomography takes
        if r.call == "fbp_ir":
            return lambda: phys.A_dagger(y, fbp=True)
        return lambda: phys.A_adjoint(y)

    def run(self, inp=None):
        with _env(self.row.env):
            return self.make_call(inp)()

    # ---- references -------------------------------------------------------------------------------------------------------
    def ref(self, inp=None):
        r = self.row
        x = (self.inp if inp is None else inp).double()
        ang, W, c = self.ang, self.W, r.circle
        if r.call == "ramp":
            return RR.ramp(x)
        if r.call in ("A", "raw_A"):
            return RR.radon_fwd(x, ang, c)
        if r.call == "At":
            return RR.radon_adj(x, ang, W, c)
        if r.call == "At_ir":
            return RR.iradon_bp(x, ang, W, c)
        if r.call == "fbp_ir":
            return RR.iradon_bp(RR.ramp(x), ang, W, c, math.pi / (2 * self.nang))
        if r.call == "fanA":
            return RR.fanbeam_fwd(x, ang, c, r.fan)
        return RR.fanbeam_adj(x, ang, W, c, r.fan)

    def oracle(self, dtype):
        """the reference's formulas (oracle/ref_ops.py) in `dtype`, for the fp32-geometry families"""
        from oracle import ref_ops as O

        r = self.row
        x, ang, W, c = self.inp.to(dtype), self.ang.to(dtype), self.W, r.circle
        if r.call == "At_ir":
            return O.tomography_At(x.transpose(-2, -1), ang, W, c, via_backprop=False)
        if r.call == "fbp_ir":
            return O.tomography_fbp(x.transpose(-2, -1), ang, W, c, via_backprop=False)
        if r.call == "fanA":
            return O.fanbeam_forward(x, ang, c, r.fan).transpose(-2, -1)
        return O.fanbeam_adjoint(x.transpose(-2, -1), ang, W, c, r.fan)

    def tol(self):
        r = self.row
        if r.call == "ramp":
            return TOL_RAMP
        if r.call in ("A", "raw_A"):
            return TOL_FWD
        # the tiled transpose's fixed-point unit is 2 A m / 2^30: its rounding grows like A^1.5 against a white-noise pixel's A^0.5
        # (1.2e-5 at A = 2048 on the H100), so beyond 360 angles the bound grows in proportion to A
        if K_TILED_A in r.kernels and self.nang > 360:
            return TOL_ADJ * self.nang / 360
        return TOL_ADJ


class _env:
    def __init__(self, kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k, _ in self.kv}
        os.environ.update(dict(self.kv))

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _per_image(got, ref, keep=None):
    """(relative L2, max |error| / max |ref|) per image (B * C), over the elements `keep` selects"""
    n = ref.shape[0] * ref.shape[1]
    d = (got.double() - ref).reshape(n, -1)
    rf = ref.reshape(n, -1)
    if keep is not None:
        k = keep.reshape(n, -1).double()
        d, rf = d * k, rf * k
    rel = d.norm(dim=1) / rf.norm(dim=1).clamp_min(1e-300)
    mx = d.abs().amax(1) / rf.abs().amax(1).clamp_min(1e-300)
    return rel, mx


def _assert_close(row, got, ref, tol, keep=None):
    rel, mx = _per_image(got, ref, keep)
    assert float(rel.max()) <= tol, f"{row.name}: image {int(rel.argmax())} relative L2 error {float(rel.max()):.3g} > {tol:g}"
    assert float(mx.max()) <= TOL_MAX, f"{row.name}: image {int(mx.argmax())} max |error| {float(mx.max()):.3g} of max |ref|"
    return dict(rel=float(rel.max()), max_abs=float(mx.max()))


def _sync(dev):
    if dev.type == "cuda":
        torch.cuda.synchronize()


def check_row(row: Row, dev: torch.device, emulated: bool = False) -> dict:
    """run one row, assert every property of the module docstring that applies to it, return the measured errors"""
    from deepinv_b200 import DinvkError, ops

    case = Case(row, dev, emulated)
    lib = ops.get_lib()
    if row.error:
        n0 = lib.dinvk_launch_count()
        try:
            case.run()
        except DinvkError as e:
            assert row.error in str(e), str(e)
        else:
            raise AssertionError(f"{row.name}: no DinvkError")
        assert lib.dinvk_launch_count() - n0 == row.launches
        return {}
    with _env(row.env):
        call = case.make_call()
        n0 = lib.dinvk_launch_count()
        got = call()
        launches = lib.dinvk_launch_count() - n0
    _sync(dev)
    got = got.cpu()
    assert launches == row.launches, f"{row.name}: {launches} launches, expected {row.launches}"
    if row.data == "nonfinite":
        return _check_nonfinite(case, got)
    ref = case.ref()
    assert tuple(got.shape) == tuple(ref.shape), (tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all(), f"{row.name}: non-finite output"
    res = {}
    if row.call in ("At_ir", "fbp_ir", "fanA", "fanAt"):
        res = _check_fp32_geometry(case, got, ref)
    else:
        res = _assert_close(row, got, ref, case.tol())
    if row.call == "raw_A":
        with _env(row.env):  # the same call on aligned memory (the tiled kernel)
            al = case._phys().A(case.inp.to(dev).contiguous()).transpose(-2, -1).cpu()
        d = float((al.double() - got.double()).norm() / al.double().norm())
        assert d < 3e-7, f"{row.name}: {d:.3g} from the same call on aligned memory"
        res["vs_aligned"] = d
    if row.data == "bitexact":
        for k in (-60, 60):
            s = 2.0 ** k
            gk = case.run(case.inp * s)
            _sync(dev)
            assert torch.equal(gk.cpu(), got * s), f"{row.name}: A^T(2^{k} y) != 2^{k} A^T(y)"
    return res


def _check_fp32_geometry(case, got, ref):
    """IRadon / fan beam: the oracle's fp32 evaluation is the yardstick (module docstring)"""
    row = case.row
    o32 = case.oracle(torch.float32)
    e_o = float((got.double() - o32.double()).norm() / o32.double().norm())
    e_k = float((got.double() - ref).norm() / ref.norm())
    e_ref = float((o32.double() - ref).norm() / ref.norm())
    assert e_o < TOL_ORACLE or e_k <= 1.15 * e_ref + 2e-7, f"{row.name}: {e_o:.3g} from the oracle, {e_k:.3g} vs its {e_ref:.3g}"
    rel, mx = _per_image(got, ref)
    assert float(mx.max()) <= 10 * TOL_ORACLE + 2 * e_ref, f"{row.name}: max |error| {float(mx.max()):.3g}"
    return dict(rel=e_k, oracle32=e_ref, vs_oracle32=e_o)


def _dilate(mask, r, image):
    m = mask.double()
    n = m.shape[0] * m.shape[1]
    if image:  # (B, C, H, W): a (2r+1)^2 neighbourhood
        return torch.nn.functional.max_pool2d(m.reshape(n, 1, *m.shape[-2:]), 2 * r + 1, 1, r).reshape(m.shape) > 0
    # sinograms (B, C, A, P): 2r+1 detector cells of the same angle
    return torch.nn.functional.max_pool1d(m.reshape(-1, 1, m.shape[-1]), 2 * r + 1, 1, r).reshape(m.shape) > 0


def _check_nonfinite(case, got):
    row = case.row
    clean = case.inp.clone()
    for a, b in case.bad:
        clean[0, 0, a, b] = 0.0
    ref = case.ref(clean)
    reach = torch.zeros(ref.shape, dtype=torch.float64)
    must = torch.zeros(ref.shape, dtype=torch.bool)
    for a, b in case.bad:
        e = torch.zeros_like(clean)
        e[0, 0, a, b] = 1.0
        w = case.ref(e)
        reach = torch.maximum(reach, w)
        must |= w > 1e-6
    near = _dilate(reach > 0, 2, image=row.call in ("At", "At_ir", "fanAt"))
    assert must.any(), row.name
    fin = torch.isfinite(got)
    assert not bool(fin[must].any()), f"{row.name}: {int(fin[must].sum())} of {int(must.sum())} reached outputs are finite"
    far = ~near
    assert bool(fin[far].all()), f"{row.name}: {int((~fin[far]).sum())} non-finite outputs far from the non-finite input"
    g = torch.where(far, got.double(), torch.zeros((), dtype=torch.float64))
    # the fp32 geometry of IRadon and fan beam sits ~1e-5 from the exact operator (_check_fp32_geometry); held to 1e-4 here
    tol = 1e-4 if row.call in ("At_ir", "fanA", "fanAt") else case.tol()
    rel, mx = _per_image(g, ref, far)
    assert float(rel.max()) <= tol, f"{row.name}: far-field relative L2 error {float(rel.max()):.3g} > {tol:g}"
    assert float(mx.max()) <= max(TOL_MAX, tol), f"{row.name}: far-field max |error| {float(mx.max()):.3g}"
    return dict(rel=float(rel.max()), max_abs=float(mx.max()), nonfinite=int((~fin).sum()), must=int(must.sum()))


# ------------------------------------------------------------------------------------------------------------------------------
# the FFT form of the ramp filter, in a child process
# ------------------------------------------------------------------------------------------------------------------------------
def install_emul(setattr_fn):
    """route deepinv_b200.ops through the host emulation of the kernel library (setattr_fn: monkeypatch.setattr or setattr)"""
    from emul_util import emul_lib

    from deepinv_b200 import _lib, ops

    lib = emul_lib()
    setattr_fn(ops, "_require_cuda", lambda *ts: torch.device("cpu"))
    setattr_fn(ops, "_stream", lambda dev: None)
    setattr_fn(ops, "get_lib", lambda: lib)
    setattr_fn(ops, "check", lambda rc: _lib.check(rc, lib))
    ops._ws_cache.clear()
    return lib


def _fft_child(emulated: bool):
    import ctypes as C

    from deepinv_b200 import ops

    if emulated:
        install_emul(setattr)
        dev = torch.device("cpu")
    else:
        dev = torch.device("cuda:0")
    lib = ops.get_lib()
    out = []
    names = set()
    for N, rows, ws in FFT_ROWS:
        g = torch.Generator().manual_seed(N * 10 + rows)
        u = torch.linspace(-1, 1, N)
        x = 30 * (1 - u * u).clamp_min(0).sqrt() + torch.randn(1, 1, rows, N, generator=g)
        xd = x.to(dev)

        def call():
            if ws:
                return ops.ramp_filter(xd)
            y = torch.empty_like(xd)
            ops.check(lib.dinvk_ramp_filter(C.c_void_p(xd.data_ptr()), C.c_void_p(y.data_ptr()), rows, N, None, 0,
                                            ops._stream(dev)))
            return y
        n0 = lib.dinvk_launch_count()
        if dev.type == "cuda":
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                y = call()
                torch.cuda.synchronize()
            kn = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
            names |= set(kn)
        else:
            y = call()
        launches = lib.dinvk_launch_count() - n0
        ref = RR.ramp(x.double())
        rel = float((y.cpu().double() - ref).norm() / ref.norm())
        out.append(dict(N=N, rows=rows, ws=ws, launches=launches, rel=rel, finite=bool(torch.isfinite(y).all())))
    # past the exact kernel's limit: N = 8193 takes the FFT form, whose padded length 32768 exceeds the row tile
    try:
        ops.ramp_filter(torch.randn(1, 1, 2, 8193, generator=torch.Generator().manual_seed(1)).to(dev))
        big = "ok"
    except Exception as e:  # noqa: BLE001  (reported to the parent, which pins the error)
        big = f"{type(e).__name__}: {e}"
    print("RAMP_FFT_JSON " + json.dumps(dict(rows=out, kernels=sorted(names), n8193=big)))


def run_fft_rows(emulated: bool) -> dict:
    """run FFT_ROWS in a child process with DINVK_RAMP_FFT=1; returns its report"""
    env = dict(os.environ, DINVK_RAMP_FFT="1")
    code = f"import sys; sys.path.insert(0, {str(HERE)!r}); import radon_path_cases as T; T._fft_child({emulated!r})"
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(HERE.parent), capture_output=True, text=True, timeout=900)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("RAMP_FFT_JSON ")]
    assert p.returncode == 0 and lines, f"child failed ({p.returncode}):\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}"
    return json.loads(lines[-1][len("RAMP_FFT_JSON "):])


def fft_launches(rows: int, ws: bool) -> int:
    """mean subtraction (with a workspace) + the row pass + the odd count's re-filtered last pair + the box response"""
    return (2 if ws else 0) + 1 + (rows & 1)


def check_fft_report(rep: dict) -> None:
    for r in rep["rows"]:
        tag = f"ramp FFT N{r['N']} rows{r['rows']} {'workspace' if r['ws'] else 'raw ABI'}"
        assert r["finite"], tag
        assert r["launches"] == fft_launches(r["rows"], r["ws"]), (tag, r["launches"])
        assert r["rel"] <= TOL_RAMP_FFT, (tag, r["rel"])
    assert rep["n8193"].startswith("DinvkError") and N8193 in rep["n8193"], rep["n8193"]
