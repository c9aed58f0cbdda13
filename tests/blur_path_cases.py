"""One case table for every launch path of the direct blur kernels (csrc/blur.cu: `blur_corr_kernel`, `blur_fold_kernel`), shared
by the H100 run (tests/test_gpu_blur_paths.py) and the host-emulated twin (tests/test_emul_blur_paths.py).

The host code runs every call as one tiled correlation (`run_corr`), plus the fold for the replicate / reflect transposes.  What
varies per call:
  * the staging of each 64 x 64 tile's halo: one TMA box (zero padding, and every tile whose halo stays inside the image) or the
    mapped cooperative loop (border tiles under circular / replicate / reflect).  The whole call takes the loop when W % 4 != 0,
    when the input is off 16-byte alignment, when a box edge would exceed 256 (filters taller than 193 rows, rows wider than about
    188 taps), under DINVK_NO_TMA_STAGING, and when only the unshifted filter layout fits the shared-memory budget;
  * `shift` = off_j mod 4 zero taps prepended to each filter row (0 .. 3, by w and the direction), which align the box;
  * the 200 KB shared-memory budget, 4 h wp + 4 (63 + h)(68 + wp) + 128 bytes (wp = w + shift rounded up to 4), past which the call
    fails with "too large"; the grid's 65535 planes, past which it fails with "grid too large".
Each row names the call, the kernels it must reach and the number of launches the host issues (A: 1; A^T: 1 for valid, circular
and constant, 2 for replicate and reflect; error rows and B = 0: none).

Every row is checked against the fp64 restatement (tests/blur_ref64.py), with s = max(1, sqrt(h w) / 31):
  * relative L2 per plane <= 1e-6 s, and per element |error| <= 64 u s abs_bound (u = 2^-24, abs_bound the operator on |k| and
    |input|): a wrong tap breaks the second by more than ten times;
  * non-finite rows: the NaN, +Inf and -Inf masks equal the restatement's exactly; finite outputs meet the bounds above;
  * on the GPU, every row also equals the same call under DINVK_NO_TMA_STAGING bit for bit (both stagings fill the same patch and
    run the same loop), and an offset input equals the aligned call bit for bit.
"""
from __future__ import annotations

import dataclasses
import math
import os
import zlib
from typing import Optional

import torch

import blur_ref64 as BR

U = 2.0 ** -24
TOL_REL, TOL_ULP = 1e-6, 64
BUDGET = 200 * 1024
K_CORR, K_FOLD = "blur_corr_kernel", "blur_fold_kernel"
NO_TMA = (("DINVK_NO_TMA_STAGING", "1"),)
PAD_CODE = {p: i for i, p in enumerate(BR.PADS)}  # include/dinvk.h: DINVK_PAD_VALID .. DINVK_PAD_CONSTANT
SAME = BR.PADS[1:]


@dataclasses.dataclass(frozen=True)
class Row:
    name: str
    call: str               # A | At | raw (ops.blur_fwd / blur_adj on a view 4 bytes past 16-byte alignment; `adj` picks which)
    B: int
    C: int
    H: int
    W: int
    h: int
    w: int
    pad: str
    FB: int = 1
    FC: int = 1
    adj: bool = False       # raw rows: the transpose
    env: tuple = ()
    data: str = "randn"     # randn | psf (cfg5: rand image, normalised rand filter) | nonfinite | infpair
    error: str = ""         # the call must raise DinvkError with this text
    emul: Optional[dict] = None  # overrides of (B, H, W) for the host emulation, on the same host branch
    gpu_only: str = ""      # why the emulation cannot check this row
    planes: tuple = ()      # batch indices checked against the restatement (empty: all)

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
# the host's geometry (csrc/blur.cu: dinvk_blur_fwd / _adj, corr_params, run_corr, tile_grid), restated
# ------------------------------------------------------------------------------------------------------------------------------
def off_j(transpose: bool, pad: str, w: int) -> int:
    if not transpose:
        return 0 if pad == "valid" else w // 2 - (w - 1)
    return -(w // 2) if pad in ("circular", "constant") else -(w - 1)


def smem_bytes(h: int, w: int, shift: int) -> int:
    wp = (w + shift + 3) & ~3
    return 4 * h * wp + 4 * (63 + h) * (68 + wp) + 128


def layout(transpose: bool, pad: str, h: int, w: int):
    """(shift, bytes) of the layout run_corr takes, or None when the filter is rejected"""
    shift = off_j(transpose, pad, w) % 4
    if smem_bytes(h, w, shift) <= BUDGET:
        return shift, smem_bytes(h, w, shift)
    if smem_bytes(h, w, 0) <= BUDGET:
        return 0, smem_bytes(h, w, 0)
    return None


def fits(h: int, w: int) -> bool:
    """the budget formula with the unshifted layout: what both directions accept, for every padding"""
    return smem_bytes(h, w, 0) <= BUDGET


def largest(shape) -> int:
    n = 1
    while fits(*shape(n + 1)):
        n += 1
    return n


N_SQ = largest(lambda n: (n, n))   # 123
N_ROW = largest(lambda n: (1, n))  # 1 x 720
N_COL = largest(lambda n: (n, 1))  # 613 x 1


def staging(row: Row, B: int, H: int, W: int) -> str:
    """'tma': the call builds a tensor map (each tile then takes the box, or the loop at a border under a mapping padding);
    'loop': every tile takes the mapped loop"""
    lay = layout(row.transpose, row.pad, row.h, row.w)
    if lay is None or row.env or row.call == "raw":
        return "loop"
    shift, _ = lay
    if shift != off_j(row.transpose, row.pad, row.w) % 4:  # the unshifted fallback
        return "loop"
    win = W - row.w + 1 if (row.transpose and row.pad == "valid") else W
    wp = (row.w + shift + 3) & ~3
    if win % 4 or 68 + wp > 256 or 63 + row.h > 256:
        return "loop"
    return "tma"


# ------------------------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------------------------
def _rows():
    R = []

    def both(tag, B, C, H, W, h, w, pads=BR.PADS, **kw):
        for pad in pads:
            for call in ("A", "At"):
                R.append(Row(f"{tag} {h}x{w} {pad} {call}", call, B, C, H, W, h, w, pad, **kw))

    # ---- tile geometry: one tile, ragged last tiles (and W % 4 != 0), 256^2 with TMA interior tiles and mapped border tiles -----
    for tag, H, W, h, w, em in (("tile 48x64", 48, 64, 7, 7, None), ("ragged 130x197", 130, 197, 5, 5, dict(H=70, W=133)),
                                ("mixed 256x256", 256, 256, 9, 9, dict(H=130, W=132))):
        both(tag, 2, 1, H, W, h, w, emul=em)
        both(tag + " no-TMA", 2, 1, H, W, h, w, env=NO_TMA, emul=em)
    # ---- shift coverage on a TMA-eligible image: w = 1 .. 8, h != w, even filters ---------------------------------------------
    for h, w in [(3, w) for w in range(1, 9)] + [(4, 7), (7, 4), (2, 5), (4, 6), (6, 6), (8, 8)]:
        both("shift 64x128", 1, 2, 64, 128, h, w)
    # ---- staging forced off: W % 4 in {1, 2, 3}, an offset input, box edges above 256 ---------------------------------------
    for W in (129, 130, 131):
        both(f"W%4={W % 4} 64x{W}", 2, 1, 64, W, 5, 5)
    for pad in BR.PADS:
        for adj in (False, True):
            R.append(Row(f"offset input 128x128 5x5 {pad} {'At' if adj else 'A'}", "raw", 2, 1, 128, 128, 5, 5, pad, adj=adj,
                         emul=dict(H=70, W=68)))
    both("box>256 512x512", 1, 1, 512, 512, 1, 301, emul=dict(H=16, W=320))
    both("box>256 512x512", 1, 1, 512, 512, 301, 1, emul=dict(H=320, W=16))
    # ---- large filters: cfg5 (planes 0 and 31), 63 x 63, the acceptance boundary ---------------------------------------------
    both("cfg5 32x1024^2", 32, 1, 1024, 1024, 31, 31, data="psf", planes=(0, 31), emul=dict(B=2, H=96, W=160))
    both("large 160x192", 1, 1, 160, 192, 63, 63, emul=dict(H=70, W=72))
    too_large = "too large"
    for h, w, H, W, em in ((N_SQ - 1, N_SQ - 1, 130, 130, dict(H=124, W=124)), (N_SQ, N_SQ, 130, 130, dict(H=124, W=124)),
                           (1, N_ROW, 6, 740, dict(H=2)), (N_COL, 1, 640, 6, dict(W=2))):
        both("accept", 1, 1, H, W, h, w, emul=em)
    for h, w, H, W in ((N_SQ + 1, N_SQ + 1, 130, 130), (1, N_ROW + 1, 6, 740), (N_COL + 1, 1, 640, 6)):
        both("reject", 1, 1, H, W, h, w, error=too_large)
    # ---- small images: 1 x 1, 1 x W, H x 1, filters larger than the image ----------------------------------------------------
    for H, W, circ, big, refl, valid in ((1, 1, (3, 3), (5, 4), (1, 1), (1, 1)), (1, 9, (3, 5), (7, 12), (1, 17), (1, 9)),
                                         (7, 1, (5, 3), (9, 5), (13, 1), (7, 1)), (3, 5, (6, 9), (8, 11), (5, 9), (3, 5))):
        tag = f"small {H}x{W}"
        both(tag, 2, 1, H, W, *circ, pads=("circular",))
        both(tag, 2, 1, H, W, *big, pads=("constant", "replicate"))
        both(tag, 2, 1, H, W, *refl, pads=("reflect",))
        both(tag, 2, 1, H, W, *valid, pads=("valid",))
    # ---- per-sample / per-channel filters ----------------------------------------------------------------------------------
    for FB, FC in ((1, 1), (3, 1), (1, 2), (3, 2)):
        both(f"broadcast FB{FB} FC{FC} 64x96", 3, 2, 64, 96, 5, 4, FB=FB, FC=FC)
    # ---- the 65535-plane grid, an empty batch ------------------------------------------------------------------------------
    slow = "65535 CTAs of 256 host threads: minutes on the emulation (its 65536-plane error row runs there)"
    both("planes 65535 8x8", 65535, 1, 8, 8, 3, 3, pads=("circular", "reflect"), gpu_only=slow)
    both("planes 65536 8x8", 32768, 2, 8, 8, 3, 3, pads=("circular", "reflect"), error="grid too large")
    both("empty batch", 0, 2, 20, 24, 3, 3)
    # ---- non-finite data: NaN / +Inf / -Inf inside a tile, on every border, on the 63 / 64 seam; TMA-eligible and loop-staged --
    for h, w in ((3, 3), (4, 6), (1, 7), (31, 31)):
        for W in (192, 190):
            both(f"non-finite 128x{W}", 2, 1, 128, W, h, w, data="nonfinite", emul=dict(H=70))
    both("opposite infinities 40x64", 1, 1, 40, 64, 3, 3, data="infpair")
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
        sh = dict(B=row.B, H=row.H, W=row.W)
        if emulated and row.emul:
            sh.update(row.emul)
        B, H, W = sh["B"], sh["H"], sh["W"]
        self.B, self.H, self.W = B, H, W
        self.planes = sorted({min(p, B - 1) for p in row.planes}) if row.planes else list(range(B))
        r = row
        self.FB = 1 if r.FB == 1 else B
        self.out_A = (B, r.C, H - r.h + 1, W - r.w + 1) if r.pad == "valid" else (B, r.C, H, W)
        in_shape = self.out_A if r.transpose else (B, r.C, H, W)
        self.out_shape = (B, r.C, H, W) if r.transpose else self.out_A
        g = torch.Generator().manual_seed(zlib.crc32(r.name.encode()))
        if r.data == "psf":
            self.inp = torch.rand(in_shape, generator=g)
            k = torch.rand(self.FB, r.FC, r.h, r.w, generator=g)
            self.k = k / k.sum(dim=(-2, -1), keepdim=True)
        else:
            self.inp = torch.randn(in_shape, generator=g)
            self.k = torch.randn(self.FB, r.FC, r.h, r.w, generator=g)
        if r.data == "nonfinite":
            self._place_nonfinite()
        elif r.data == "infpair":  # footprints 3 columns apart: they overlap
            self.inp[0, 0, 20, 30], self.inp[0, 0, 21, 32] = float("inf"), float("-inf")

    def _place_nonfinite(self):
        """in each plane: inside a tile, on row 0, column 0, the last row and the last column, and on the 63 / 64 column seam"""
        Hi, Wi = self.inp.shape[-2:]
        locs = [(Hi // 3, Wi // 2 + 5), (0, Wi // 3), (Hi // 2, 0), (Hi - 1, (2 * Wi) // 3), ((2 * Hi) // 3, Wi - 1),
                (Hi // 4, 63), (Hi // 4 + 9, 64)]
        vals = (float("nan"), float("inf"), float("-inf"))
        for b in range(self.inp.shape[0]):
            for n, (p, q) in enumerate(locs):
                if p < Hi and q < Wi:
                    self.inp[b, 0, p, q] = vals[(n + b) % 3]

    # ---- the call under test ----------------------------------------------------------------------------------------------
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
                return lambda: ops.blur_adj(xv, k, code, self.H, self.W)
            return lambda: ops.blur_fwd(xv, k, code)
        phys = dinv.physics.Blur(filter=k, padding=r.pad, device=self.dev)
        return (lambda: phys.A_adjoint(x)) if r.transpose else (lambda: phys.A(x))

    def run(self, env=None):
        with _env(self.row.env if env is None else env):
            return self.make_call()()

    # ---- references -------------------------------------------------------------------------------------------------------
    def ref(self):
        """(restatement, abs_bound) on the checked planes"""
        r = self.row
        pl = self.planes
        inp, k = self.inp[pl].double(), (self.k[pl] if self.FB > 1 else self.k).double()
        call = "At" if r.transpose else "A"
        return BR.apply(call, inp, k, r.pad, self.H, self.W), BR.abs_bound(call, inp, k, r.pad, self.H, self.W)

    def scale(self):
        return max(1.0, math.sqrt(self.row.h * self.row.w) / 31)


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


def _sync(dev):
    if dev.type == "cuda":
        torch.cuda.synchronize()


def _compare(row, case, got, ref, bound):
    """the bounds of the module docstring on the finite outputs; exact non-finite masks"""
    g = got.double()
    for name, f in (("NaN", torch.isnan), ("+Inf", lambda t: t == float("inf")), ("-Inf", lambda t: t == float("-inf"))):
        a, b = f(g), f(ref)
        assert torch.equal(a, b), f"{row.name}: {name} mask differs at {int((a ^ b).sum())} outputs ({int(b.sum())} expected)"
    fin = torch.isfinite(ref)
    zero = torch.zeros((), dtype=torch.float64)
    d = torch.where(fin, g - ref, zero)
    rf = torch.where(fin, ref, zero)
    n = ref.shape[0] * ref.shape[1]
    rel = d.reshape(n, -1).norm(dim=1) / rf.reshape(n, -1).norm(dim=1).clamp_min(1e-300)
    s = case.scale()
    assert float(rel.max()) <= TOL_REL * s, f"{row.name}: plane {int(rel.argmax())} relative L2 {float(rel.max()):.3g} > {TOL_REL * s:.3g}"
    ulps = torch.where(fin, d.abs() / (U * bound).clamp_min(1e-300), zero)
    worst = float(ulps.max())
    assert worst <= TOL_ULP * s, f"{row.name}: |error| = {worst:.1f} u abs_bound > {TOL_ULP * s:.1f} (at {tuple(int(i) for i in (ulps == worst).nonzero()[0])})"
    return dict(rel=float(rel.max()), ulps=worst, nonfinite=int((~fin).sum()))


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
    res["staging"] = staging(row, case.B, case.H, case.W)
    return res


def _same_nan(a, b):
    """bit-for-bit equality where NaN payloads may differ"""
    both = torch.isnan(a) & torch.isnan(b)
    return torch.equal(torch.where(both, 0.0, a), torch.where(both, 0.0, b))
