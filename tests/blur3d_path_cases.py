"""One case table for every launch path of the 3-D blur kernels (csrc/blur.cu: `blur3d_corr_kernel`, `blur3d_fold_kernel`), shared
by the H100 run (tests/test_gpu_blur3d.py) and the host-emulated twin (tests/test_emul_blur3d_paths.py).

The host code runs every call as one tiled 3-D correlation (`run_corr3d`), plus the fold for the replicate / reflect transposes.
What varies per call:
  * the staging of each plane's 64 x 64 tile + halo: one TMA box (zero padding, and every tile whose halo stays inside the plane)
    or the mapped cooperative loop, as in 2-D.  The whole call takes the loop when W % 4 != 0, when the input is off 16-byte
    alignment, when a box edge would exceed 256, under DINVK_NO_TMA_STAGING, and when only the unshifted filter layout fits;
  * `shift` = off_j mod 4 zero taps prepended to each filter row (0 .. 3, by w and the direction);
  * the layout: B3_ZT = 4 output planes per CTA with two patch buffers, else one buffer, else one plane (one filter slice and one
    patch, the 2-D kernel's footprint and limit: 4 h wp + 4 (63 + h)(68 + wp) + 128 bytes <= 200 KB), past which the call fails
    with "too large"; the depth of the filter is not limited (slices stream through a ring);
  * the depth walk: planes outside the volume under zero padding are skipped, the others map by the padding rule at both ends;
  * the grid's 65535 (b, c) volumes, past which the call fails with "grid too large".
Each row names the call, the kernels it must reach and the number of launches (A: 1; A^T: 1 for valid, circular and constant, 2
for replicate and reflect; error rows and B = 0: none).

Every row is checked against the fp64 restatement (tests/blur3d_ref64.py) with the 2-D bounds of tests/blur_path_cases.py and
s = max(1, sqrt(d h w / 961)); non-finite masks must match exactly; on the GPU the TMA and loop stagings agree bit for bit and an
offset input equals the aligned call.
"""
from __future__ import annotations

import dataclasses
import math
import zlib
from typing import Optional

import torch

import blur3d_ref64 as BR3
from blur_path_cases import NO_TMA, PAD_CODE, _compare, _env, _same_nan, _sync  # noqa: F401  (the 2-D table's checks)

BUDGET = 200 * 1024
ZT = 4
K_CORR, K_FOLD = "blur3d_corr_kernel", "blur3d_fold_kernel"
PADS = BR3.PADS


@dataclasses.dataclass(frozen=True)
class Row:
    name: str
    call: str               # A | At | raw (ops.blur3d_fwd / blur3d_adj on a view 4 bytes past 16-byte alignment; `adj` picks which)
    B: int
    C: int
    D: int
    H: int
    W: int
    d: int
    h: int
    w: int
    pad: str
    FB: int = 1
    FC: int = 1
    adj: bool = False
    env: tuple = ()
    data: str = "randn"     # randn | psf (rand volume, normalised rand filter) | nonfinite
    error: str = ""         # the call must raise DinvkError with this text
    emul: Optional[dict] = None  # overrides of (B, C, D, H, W) for the host emulation, on the same host branch
    gpu_only: str = ""

    @property
    def transpose(self):
        return self.call == "At" or (self.call == "raw" and self.adj)

    @property
    def kernels(self):
        if self.error or self.B == 0:
            return ()
        return (K_CORR, K_FOLD) if self.transpose and self.pad in ("replicate", "reflect") else (K_CORR,)

    @property
    def launches(self):
        return len(self.kernels)


# ------------------------------------------------------------------------------------------------------------------------------
# the host's geometry (csrc/blur.cu: dinvk_blur3d_fwd / _adj, run_corr3d), restated
# ------------------------------------------------------------------------------------------------------------------------------
def off_j(transpose: bool, pad: str, w: int) -> int:
    if not transpose:
        return 0 if pad == "valid" else w // 2 - (w - 1)
    return -(w // 2) if pad in ("circular", "constant") else -(w - 1)


def smem_bytes(zt: int, nbuf: int, h: int, w: int, shift: int) -> int:
    wp = (w + shift + 3) & ~3
    return (zt + nbuf - 1) * 4 * h * wp + nbuf * (4 * (63 + h) * (68 + wp) + 128)


def layout(transpose: bool, pad: str, h: int, w: int):
    """(zt, nbuf, shift) of the layout run_corr3d takes, or None when the filter is rejected"""
    shift = off_j(transpose, pad, w) % 4
    for zt, nbuf in ((ZT, 2), (ZT, 1), (1, 1)):
        if smem_bytes(zt, nbuf, h, w, shift) <= BUDGET:
            return zt, nbuf, shift
    if shift and smem_bytes(1, 1, h, w, 0) <= BUDGET:
        return 1, 1, 0
    return None


def largest(zt, nbuf) -> int:
    """the largest square slice the layout takes in both directions for every padding"""
    n = 1
    while all(smem_bytes(zt, nbuf, n + 1, n + 1, s) <= BUDGET for s in range(4)):
        n += 1
    return n


N_DB, N_SB, N_ONE = largest(ZT, 2), largest(ZT, 1), 123  # 123: the 2-D limit, unshifted


def staging(row: Row, W: int) -> str:
    lay = layout(row.transpose, row.pad, row.h, row.w)
    if lay is None or row.env or row.call == "raw":
        return "loop"
    zt, nbuf, shift = lay
    if shift != off_j(row.transpose, row.pad, row.w) % 4:
        return "loop"
    win = W - row.w + 1 if (row.transpose and row.pad == "valid") else W
    wp = (row.w + shift + 3) & ~3
    return "loop" if (win % 4 or 68 + wp > 256 or 63 + row.h > 256) else "tma"


# ------------------------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------------------------
def _rows():
    R = []

    def both(tag, B, C, D, H, W, d, h, w, pads=PADS, **kw):
        for pad in pads:
            for call in ("A", "At"):
                R.append(Row(f"{tag} {d}x{h}x{w} {pad} {call}", call, B, C, D, H, W, d, h, w, pad, **kw))

    # ---- staging: one tile; 256^2 planes whose interior tiles take the box and border tiles the loop; no TMA ------------------
    both("tile 6x48x64", 2, 1, 6, 48, 64, 3, 5, 5)
    both("tile 6x48x64 no-TMA", 2, 1, 6, 48, 64, 3, 5, 5, env=NO_TMA)
    both("mixed 5x256x256", 1, 1, 5, 256, 256, 3, 9, 9, emul=dict(H=130, W=132))
    both("mixed 5x256x256 no-TMA", 1, 1, 5, 256, 256, 3, 9, 9, env=NO_TMA, emul=dict(H=130, W=132))
    # ---- every shift in both directions (w = 1 .. 8), even extents -----------------------------------------------------------
    for w in range(1, 9):
        both("shift 5x64x128", 1, 1, 5, 64, 128, 2, 3, w, pads=("circular", "replicate"), emul=dict(W=68))
    # ---- the depth walk: both ends under each padding, D not a multiple of 4, D < d, D = 1, deep filters (streamed slices) -----
    both("depth 6x40x44", 2, 1, 6, 40, 44, 5, 3, 3)
    both("depth 7x40x44", 1, 1, 7, 40, 44, 4, 3, 2)
    both("D<d 2x20x24", 2, 1, 2, 20, 24, 5, 3, 3, pads=("circular", "replicate", "constant"))
    both("D=1 1x20x24", 2, 1, 1, 20, 24, 3, 3, 3, pads=("circular", "replicate", "constant"))
    both("D=1 1x20x24", 2, 1, 1, 20, 24, 1, 3, 3)
    both("deep 40x20x24", 1, 1, 40, 20, 24, 33, 3, 3)
    both("too small 2x20x24", 1, 1, 2, 20, 24, 5, 3, 3, pads=("valid", "reflect"), error="blur3d")
    # ---- W % 4 != 0, box edges above 256, an offset input --------------------------------------------------------------------
    both("W%4=1 5x64x129", 1, 1, 5, 64, 129, 3, 5, 5, pads=("circular", "constant", "valid"), emul=dict(H=20, W=69))
    both("box>256 3x8x320", 1, 1, 3, 8, 320, 1, 1, 201, pads=("circular", "valid"))
    for pad in PADS:
        for adj in (False, True):
            R.append(Row(f"offset input 5x64x64 3x5x5 {pad} {'At' if adj else 'A'}", "raw", 2, 1, 5, 64, 64, 3, 5, 5, pad, adj=adj))
    # ---- layouts: the largest slice of each, one past it (the next layout), the 2-D limit and past it ------------------------
    for n, zd in ((N_DB, 3), (N_DB + 1, 3), (N_SB, 2), (N_SB + 1, 2), (N_ONE, 2)):
        both(f"slice {n}", 1, 1, 6, 130, 130, 2, n, n, pads=("circular", "valid"), emul=dict(D=zd, H=n + 2, W=n + 3))
    both("reject", 1, 1, 3, 130, 130, 2, N_ONE + 1, N_ONE + 1, pads=("circular", "valid"), error="too large")
    # ---- microscopy size: 15^3 PSF on 64 planes of 256^2, one volume -----------------------------------------------------------
    both("psf 64x256x256", 1, 1, 64, 256, 256, 15, 15, 15, pads=("circular", "valid"), data="psf",
         gpu_only="15^3 taps per voxel over 4M voxels: hours on the emulation")
    # ---- per-sample / per-channel filters --------------------------------------------------------------------------------------
    for FB, FC in ((1, 1), (3, 1), (1, 2), (3, 2)):
        both(f"broadcast FB{FB} FC{FC} 5x20x36", 3, 2, 5, 20, 36, 3, 5, 4, FB=FB, FC=FC, pads=("circular", "reflect", "valid"))
    # ---- the 65535-volume grid, an empty batch ---------------------------------------------------------------------------------
    slow = "65535 volumes of 256 host threads per CTA: minutes on the emulation (its 65536-volume error row runs there)"
    both("volumes 65535 2x8x8", 65535, 1, 2, 8, 8, 1, 3, 3, pads=("circular", "reflect"), gpu_only=slow)
    both("volumes 65536 2x8x8", 32768, 2, 2, 8, 8, 1, 3, 3, pads=("circular", "reflect"), error="grid too large")
    both("empty batch", 0, 2, 4, 20, 24, 3, 3, 3)
    # ---- NaN / +Inf / -Inf voxels: inside, on every face, on the 63 / 64 column seam; TMA-eligible and loop-staged -------------
    for (d, h, w) in ((3, 3, 3), (2, 4, 6), (5, 1, 7)):
        for W in (128, 126):
            both(f"non-finite 7x70x{W}", 2, 1, 7, 70, W, d, h, w, data="nonfinite", emul=dict(H=40))
    names = [r.name for r in R]
    assert len(names) == len(set(names)), [n for n in names if names.count(n) > 1]
    return R


ROWS = _rows()


# ------------------------------------------------------------------------------------------------------------------------------
# inputs, calls, references
# ------------------------------------------------------------------------------------------------------------------------------
class Case:
    def __init__(self, row: Row, dev: torch.device, emulated: bool = False):
        self.row, self.dev = row, dev
        sh = dict(B=row.B, C=row.C, D=row.D, H=row.H, W=row.W)
        if emulated and row.emul:
            sh.update(row.emul)
        B, C, D, H, W = (sh[k] for k in "BCDHW")
        self.B, self.C, self.D, self.H, self.W = B, C, D, H, W
        self.planes = list(range(B)) if B <= 4 else [0, B - 1]
        r = row
        self.FB = 1 if r.FB == 1 else B
        self.out_A = (B, C, D - r.d + 1, H - r.h + 1, W - r.w + 1) if r.pad == "valid" else (B, C, D, H, W)
        valid_in = all(n >= 1 for n in self.out_A[2:])
        in_shape = (self.out_A if valid_in else (B, C, 1, 1, 1)) if r.transpose else (B, C, D, H, W)
        self.out_shape = (B, C, D, H, W) if r.transpose else self.out_A
        g = torch.Generator().manual_seed(zlib.crc32(r.name.encode()))
        if r.data == "psf":
            self.inp = torch.rand(in_shape, generator=g)
            k = torch.rand(self.FB, r.FC, r.d, r.h, r.w, generator=g)
            self.k = k / k.sum(dim=(-3, -2, -1), keepdim=True)
        else:
            self.inp = torch.randn(in_shape, generator=g)
            self.k = torch.randn(self.FB, r.FC, r.d, r.h, r.w, generator=g)
        if r.data == "nonfinite":
            self._place_nonfinite()

    def _place_nonfinite(self):
        """per volume: inside, on the first and last plane, row 0, column 0, the last row and column, and the 63 / 64 seam"""
        Di, Hi, Wi = self.inp.shape[-3:]
        locs = [(Di // 2, Hi // 3, Wi // 2 + 5), (0, Hi // 2, Wi // 3), (Di - 1, Hi // 4, Wi // 4), (Di // 3, 0, Wi // 3),
                (Di // 2, Hi // 2, 0), (Di // 2, Hi - 1, (2 * Wi) // 3), (1 % Di, (2 * Hi) // 3, Wi - 1), (Di // 2, Hi // 4, 63),
                (Di // 2, Hi // 4 + 9, 64)]
        vals = (float("nan"), float("inf"), float("-inf"))
        for b in range(self.inp.shape[0]):
            for n, (z, p, q) in enumerate(locs):
                if q < Wi:
                    self.inp[b, 0, z, p, q] = vals[(n + b) % 3]

    def make_call(self, inp=None):
        import deepinv_b200 as dinv
        from deepinv_b200 import ops

        r = self.row
        x = (self.inp if inp is None else inp).to(self.dev)
        k = self.k.to(self.dev)
        if r.call == "raw":
            flat = torch.zeros(x.numel() + 1, device=self.dev)
            flat[1:] = x.reshape(-1)
            xv = flat[1:].view(x.shape)
            assert xv.data_ptr() % 16 == 4
            code = PAD_CODE[r.pad]
            if r.adj:
                return lambda: ops.blur3d_adj(xv, k, code, self.D, self.H, self.W)
            return lambda: ops.blur3d_fwd(xv, k, code)
        phys = dinv.physics.Blur(filter=k, padding=r.pad, device=self.dev)
        if r.transpose:
            return lambda: ops.blur3d_adj(x, k, PAD_CODE[r.pad], self.D, self.H, self.W) if r.error else phys.A_adjoint(x)
        return lambda: phys.A(x)

    def run(self, env=None):
        with _env(self.row.env if env is None else env):
            return self.make_call()()

    def ref(self):
        r = self.row
        pl = self.planes
        inp, k = self.inp[pl].double(), (self.k[pl] if self.FB > 1 else self.k).double()
        call = "At" if r.transpose else "A"
        return BR3.apply(call, inp, k, r.pad, self.D, self.H, self.W), BR3.abs_bound(call, inp, k, r.pad, self.D, self.H, self.W)

    def scale(self):
        return max(1.0, math.sqrt(self.row.d * self.row.h * self.row.w / 961))


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
        assert lib.dinvk_launch_count() - n0 == 0
        return {}
    with _env(row.env):
        call = case.make_call()
        n0 = lib.dinvk_launch_count()
        got = call()
        launches = lib.dinvk_launch_count() - n0
    _sync(dev)
    assert launches == row.launches, f"{row.name}: {launches} launches, expected {row.launches}"
    assert tuple(got.shape) == case.out_shape, (tuple(got.shape), case.out_shape)
    if case.B == 0:
        return {}
    got = got.cpu()
    ref, bound = case.ref()
    res = _compare(row, case, got[case.planes], ref, bound)
    if row.data in ("randn", "psf"):
        assert res["nonfinite"] == 0, row.name
    if dev.type == "cuda" and not row.env:  # the TMA box and the mapped loop stage the same patch values
        alt = case.run(NO_TMA)
        _sync(dev)
        assert torch.equal(alt.cpu(), got) or _same_nan(alt.cpu(), got), f"{row.name}: TMA and mapped staging differ"
    if row.call == "raw":  # the same call on aligned memory
        al = Row(**{**dataclasses.asdict(row), "call": "At" if row.adj else "A"})
        c2 = Case(al, dev, emulated)
        c2.inp, c2.k = case.inp, case.k
        aligned = c2.run().cpu()
        assert torch.equal(aligned, got) or _same_nan(aligned, got), f"{row.name}: differs from the aligned call"
    res["staging"] = staging(row, case.W)
    res["layout"] = layout(row.transpose, row.pad, row.h, row.w)
    return res
