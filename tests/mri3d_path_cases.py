"""One case table for every launch path of `dinvk_spectral3d`, shared by the H100 run (tests/test_gpu_mri3d.py) and the host-emulated
twin (tests/test_emul_mri3d_paths.py).

The 3-D entry runs each axis as a pass of the 2-D family over a view of the volume (csrc/spectral.cu): the depth pass is a column
pass over (D, H*W), the H pass a column pass over the B*D slices, the W pass a row pass over (D*H, W).  Each pass picks its kernel
from its own length and alignment: the power-of-two fast kernels (rows N = 64 .. 1024, columns N = 128 .. 1024), the generic
mixed-radix tile passes, and, when any axis has a prime factor above 5, the O(N²) axis DFT on all three axes between elementwise
passes.  Each row names its family, its launch count and the kernels it must launch (the GPU census checks the last).

Every row is checked against the fp64 contract (tests/mri3d_ref64.py) with the bounds of tests/spectral_path_cases.py:
  * relative L2 error per volume (per volume and coil for coil_mode 1) < 1e-5;
  * max |error| per volume <= 1e-5 * max |ref| of that volume;
  * off the O(N²) path: error <= max(4 x the error of torch's own fp32 evaluation of the same contract, 5e-7);
  * the exact zero pattern of a 0/1-masked `A`;
  * rows whose operands sit off 16-byte alignment also agree within 3e-6 with the same call on aligned copies.
"""
from __future__ import annotations

import dataclasses
import zlib
from typing import Optional

import torch

import mri3d_ref64 as S

TOL = 1e-5
FLOOR = 5e-7
FWD, ADJ, FUSED, ELEM = (1, 0), (0, 1), (1, 1), (0, 0)
K_PASS, K_FAST, K_DFT, K_COIL = "spectral_pass_kernel", "spectral_fast_kernel", "dft_axis_naive_kernel", "coil_combine_kernel"
LIBRARY_KERNELS = (K_PASS, K_FAST, K_DFT, K_COIL)


@dataclasses.dataclass(frozen=True)
class Row:
    name: str
    shape: tuple            # (B, D, H, W); B counts batch samples (coil volumes are B * ncoil)
    op: tuple               # (fwd, inv)
    gmode: int
    mask: str               # none | full | shared | weighted | cplx
    path: str               # fast | tile | naive | elem
    kernels: tuple          # the library kernels the call launches (all of them, nothing else)
    centered: bool = True
    epi: bool = False
    prox: bool = False
    cb: bool = False
    ncoil: int = 0
    coil_mode: int = 0
    maps: str = "shared"    # shared | per
    e0: float = 1.0
    offset: int = 0
    emul: Optional[tuple] = None  # smaller (B, D, H, W) for the host emulation, on the same path with the same launch count

    @property
    def launches(self) -> int:
        if self.shape[0] == 0:
            return 0
        if self.path == "elem":
            return 1
        red = 1 if self.coil_mode >= 2 else 0
        if self.path == "naive":  # prologue, 3 axis DFTs per direction, the middle multiplier, epilogue / coil reduction
            return 9 if self.op == FUSED else 5
        return (5 if self.op == FUSED else 3) + red


def _k(path, coil_mode=0, fast=False, generic=True):
    ks = {"naive": (K_PASS, K_DFT), "elem": (K_PASS,)}.get(path)
    if ks is None:
        ks = ((K_FAST,) if fast else ()) + ((K_PASS,) if generic else ())
    return ks + ((K_COIL,) if coil_mode >= 2 else ())


def _rows():
    R = []

    def row(name, shape, op, gmode, mask, path, kernels, **kw):
        R.append(Row(name, shape, op, gmode, mask, path, kernels, **kw))

    # ---- kernel families per axis ----------------------------------------------------------------------------------------------
    # 128 x 64 x 64: depth on the fast column kernel, H generic (fast columns start at 128), W on the fast row kernel
    # 64 x 256 x 256: depth generic, H and W fast (workload (c) of tools/mri3d_bench.py)
    # 160 x 32 x 48: radix-5 depth, every pass generic; 15 x 27 x 25: odd smooth sizes, centred and plain
    # 5 x 17 x 11 (the reference's test size) and 7 x 16 x 16 (a prime depth): the O(N²) path
    fams = [("p2 128x64x64", (2, 128, 64, 64), "tile", _k("tile", fast=True), (1, 128, 8, 64)),
            ("p2 64x256x256", (1, 64, 256, 256), "tile", _k("tile", fast=True), (1, 2, 256, 64)),
            ("radix5 160x32x48", (1, 160, 32, 48), "tile", _k("tile"), (1, 160, 4, 12)),
            ("odd 15x27x25", (2, 15, 27, 25), "tile", _k("tile"), None),
            ("prime 5x17x11", (2, 5, 17, 11), "naive", _k("naive"), None),
            ("prime depth 7x16x16", (2, 7, 16, 16), "naive", _k("naive"), None)]
    for f, shape, path, ks, em in fams:
        row(f"{f} A", shape, FWD, S.G_MASK, "full", path, ks, emul=em)
        row(f"{f} At", shape, ADJ, S.G_MASK, "full", path, ks, emul=em)
        row(f"{f} AtA", shape, FUSED, S.G_SQ, "full", path, ks, emul=em)
        row(f"{f} prox shared", shape, FUSED, S.G_INV_SQ_PLUS_C, "shared", path, ks, prox=True, emul=em)
    for cen in (True, False):
        c = "centred" if cen else "plain"
        row(f"odd 9x15x25 A {c}", (1, 9, 15, 25), FWD, S.G_MASK, "full", "tile", _k("tile"), centered=cen)
        row(f"odd 9x15x25 AtA {c}", (1, 9, 15, 25), FUSED, S.G_SQ, "weighted", "tile", _k("tile"), centered=cen)
        row(f"prime 3x7x11 AtA {c}", (1, 3, 7, 11), FUSED, S.G_SQ, "weighted", "naive", _k("naive"), centered=cen)
    # ---- coils: modes 1 / 2 / 3, shared and per-sample maps, one coil, on each family ------------------------------------------
    cfams = [("tile", (2, 6, 10, 12), 4, None), ("naive", (1, 5, 17, 11), 15, None), ("fast", (1, 128, 16, 64), 3, (1, 128, 4, 64))]
    for fam, shape, N, em in cfams:
        path = "naive" if fam == "naive" else "tile"
        for maps in ("shared", "per"):
            for mode in (1, 2, 3):
                ks = _k(path, mode, fast=fam == "fast")
                row(f"coils {fam} {N} {maps} mode {mode}", shape, FWD if mode == 1 else ADJ, S.G_MASK, "full", path, ks, ncoil=N,
                    coil_mode=mode, maps=maps, e0=0.7 if mode == 2 else 1.0, emul=em)
        for mode in (1, 2, 3):
            ks = _k(path, mode, fast=fam == "fast")
            row(f"coils {fam} 1 mode {mode}", shape, FWD if mode == 1 else ADJ, S.G_MASK, "shared", path, ks, ncoil=1,
                coil_mode=mode, maps="per", emul=em)
    # ---- no maps, a (B,2,N,D,H,W) stack (the coils of a k-space tensor through V / V^T): every op, mask of the sample ----------
    for fam, shape, ks, em in (("tile", (2, 6, 10, 12), _k("tile"), None), ("naive", (2, 5, 7, 13), _k("naive"), None),
                               ("fast", (1, 128, 16, 64), _k("tile", fast=True), (1, 128, 4, 64))):
        path = "naive" if fam == "naive" else "tile"
        row(f"stack {fam} 3 A", shape, FWD, S.G_MASK, "full", path, ks, ncoil=3, emul=em)
        row(f"stack {fam} 3 At", shape, ADJ, S.G_MASK, "shared", path, ks, ncoil=3, emul=em)
        row(f"stack {fam} 3 fused g3 c_batch", shape, FUSED, S.G_INV_SQ_PLUS_C, "weighted", path, ks, ncoil=3, epi=True, cb=True,
            emul=em)
        row(f"stack {fam} 3 V", shape, FWD, S.G_NONE, "none", path, ks, ncoil=3, emul=em)
    # ---- mixed axes: one axis with a prime factor above 5 takes the O(N²) DFT, the others keep their tile passes ---------------
    row("mixed 7x256x256 A", (1, 7, 256, 256), FWD, S.G_MASK, "full", "naive", (K_PASS, K_FAST, K_DFT), emul=(1, 7, 256, 64))
    row("mixed 7x256x256 AtA", (1, 7, 256, 256), FUSED, S.G_SQ, "full", "naive", (K_PASS, K_FAST, K_DFT), emul=(1, 7, 256, 64))
    row("mixed 64x11x128 At", (2, 64, 11, 128), ADJ, S.G_MASK, "full", "naive", (K_PASS, K_FAST, K_DFT), emul=(1, 8, 11, 128))
    row("mixed 160x48x13 coils mode 2", (1, 160, 48, 13), ADJ, S.G_MASK, "full", "naive", _k("naive", 2), ncoil=3, coil_mode=2,
        emul=(1, 160, 4, 13))
    # ---- every gmode, c_batch and the full epilogue on each family --------------------------------------------------------------
    gfams = [("tile", (2, 6, 10, 12), _k("tile"), None), ("naive", (2, 5, 7, 13), _k("naive"), None),
             ("fast", (1, 128, 16, 64), _k("tile", fast=True), (1, 128, 4, 64))]
    for fam, shape, ks, em in gfams:
        path = "naive" if fam == "naive" else "tile"
        f = f"gmodes {fam}"
        for gm, m in ((S.G_MASK, "full"), (S.G_SQ, "weighted"), (S.G_INV_SQ_PLUS_C, "weighted"), (S.G_PINV, "weighted"),
                      (S.G_CMUL, "cplx"), (S.G_CMUL_CONJ, "cplx")):
            row(f"{f} fused g{gm}", shape, FUSED, gm, m, path, ks, epi=True, centered=gm < S.G_CMUL, emul=em)
        row(f"{f} A g1", shape, FWD, S.G_MASK, "full", path, ks, epi=True, emul=em)
        row(f"{f} At g4", shape, ADJ, S.G_PINV, "weighted", path, ks, epi=True, emul=em)
        row(f"{f} fused g3 c_batch", shape, FUSED, S.G_INV_SQ_PLUS_C, "weighted", path, ks, cb=True, prox=True, emul=em)
    # ---- elementwise only (fwd = inv = 0), every gmode ------------------------------------------------------------------------
    for gm, m in ((S.G_NONE, "none"), (S.G_MASK, "full"), (S.G_SQ, "weighted"), (S.G_INV_SQ_PLUS_C, "weighted"),
                  (S.G_PINV, "weighted"), (S.G_CMUL, "cplx"), (S.G_CMUL_CONJ, "cplx")):
        row(f"elementwise g{gm}", (3, 4, 9, 7), ELEM, gm, m, "elem", _k("elem"), epi=True)
    # ---- operands 4 or 8 bytes off 16-byte alignment leave the fast kernels -----------------------------------------------------
    for off in (1, 2):
        a = f"align +{off}"
        for nm, op, gm in (("A", FWD, S.G_MASK), ("At", ADJ, S.G_MASK), ("AtA", FUSED, S.G_SQ)):
            row(f"{a} {nm}", (1, 128, 16, 64), op, gm, "full", "tile", _k("tile"), epi=True, offset=off, emul=(1, 128, 4, 64))
        row(f"{a} coils mode 2", (1, 6, 10, 12), ADJ, S.G_MASK, "full", "tile", _k("tile", 2), ncoil=3, coil_mode=2, maps="per",
            offset=off)
    # ---- empty batch: no launch --------------------------------------------------------------------------------------------------
    row("empty A", (0, 4, 8, 8), FWD, S.G_MASK, "shared", "tile", ())
    row("empty coils mode 2", (0, 4, 8, 8), ADJ, S.G_MASK, "shared", "tile", (), ncoil=3, coil_mode=2)
    names = [r.name for r in R]
    assert len(names) == len(set(names))
    return R


ROWS = _rows()


def _mask(kind, B, D, H, W, g):
    """(tensor, (sb, sc, sh), complex?, binary?) in the ABI's addressing (dinvk.h, dinvk_spectral3d)"""
    V = D * H * W
    if kind == "full":
        return (torch.rand(B, 2, D, H, W, generator=g) > 0.5).float(), (2 * V, V, W), False, True
    if kind == "shared":
        return (torch.rand(1, 2, D, H, W, generator=g) > 0.5).float(), (0, V, W), False, True
    if kind == "weighted":
        t = (0.05 + 0.95 * torch.rand(B, 2, D, H, W, generator=g)) * (torch.rand(B, 2, D, H, W, generator=g) > 0.3).float()
        t.view(-1)[::97] = 3e-6
        return t, (2 * V, V, W), False, False
    if kind == "cplx":
        return torch.randn(B, D, H, W, 2, generator=g), (V, 0, W), True, False
    raise ValueError(kind)


class Case:
    def __init__(self, row: Row, dev: torch.device, shape=None):
        self.row, self.dev = row, dev
        B, D, H, W = self.shape = tuple(shape or row.shape)
        self.g = g = torch.Generator().manual_seed(zlib.crc32(row.name.encode()))
        nc = max(row.ncoil, 1)
        self.nc = nc
        stack = row.coil_mode == 0 and nc > 1  # a plain (B,2,N,D,H,W) stack of volumes, no maps
        src = (B, 2, nc, D, H, W) if row.coil_mode >= 2 or stack else (B, 2, D, H, W)
        self.out_shape = {1: (B, 2, nc, D, H, W), 2: (B, 2, D, H, W), 3: (B, 1, D, H, W)}.get(row.coil_mode, src)
        c = {"p0": torch.randn(src, generator=g)}
        if row.epi or row.prox:
            c["p1"] = torch.randn(src, generator=g)
        if row.epi:
            c["q0"] = torch.randn(self.out_shape, generator=g)
            c["q1"] = torch.randn(self.out_shape, generator=g)
        self.cpu = c
        self.binary = False
        if row.gmode != S.G_NONE:
            self.mt, self.strides, self.cplx, self.binary = _mask(row.mask, max(B, 1), D, H, W, g)
        self.scal = dict(a0=0.5 if row.epi else 1.0, a1=-1.5 if row.epi else (1 / 0.7 if row.prox else 0.0),
                         e0=2.0 if row.epi else row.e0, e1=0.25 if row.epi else 0.0, e2=-0.75 if row.epi else 0.0, c=1 / 0.7)
        self.cb = (torch.rand(B, generator=g) + 0.5) if row.cb else None
        self.maps = None
        if row.coil_mode:
            mp = torch.randn(1 if row.maps == "shared" else B, nc, D, H, W, generator=g, dtype=torch.complex64)
            self.maps = (mp / mp.abs().pow(2).sum(1, keepdim=True).sqrt()).contiguous()

    def _place(self, t, offset):
        if offset == 0:
            return t.to(self.dev).contiguous()
        flat = torch.zeros(t.numel() + offset, dtype=t.dtype, device=self.dev)
        flat[offset:] = t.reshape(-1).to(self.dev)
        return flat[offset:].view(t.shape)

    def make_call(self, offset=None):
        from deepinv_b200 import ops

        r = self.row
        offset = r.offset if offset is None else offset
        B, D, H, W = self.shape
        d = {k: self._place(v, offset if k != "q1" else 0) for k, v in self.cpu.items()}
        kw = dict(fwd=bool(r.op[0]), inv=bool(r.op[1]), centered=r.centered, gmode=r.gmode, c=self.scal["c"],
                  a0=self.scal["a0"], a1=self.scal["a1"], e0=self.scal["e0"], e1=self.scal["e1"], e2=self.scal["e2"],
                  p1=d.get("p1"), q0=d.get("q0"), q1=d.get("q1"))
        if r.gmode != S.G_NONE:
            sb, sc, sh = self.strides
            kw["mask"] = ops.MaskSpec(self._place(self.mt, offset), sb, sc, sh, self.cplx)
        if self.cb is not None:
            kw["c_batch"] = self.cb.to(self.dev)
        if r.coil_mode:
            kw.update(ncoil=self.nc, coil_mode=r.coil_mode, coil_maps=self._place(self.maps, offset))
        return lambda: ops.spectral3d(d["p0"], D, H, W, **kw)

    def ref(self, dtype=torch.float64):
        r = self.row
        B, D, H, W = self.shape
        c = self.cpu
        kw = dict(fwd=r.op[0], inv=r.op[1], centered=r.centered, gmode=r.gmode, p1=c.get("p1"), q0=c.get("q0"), q1=c.get("q1"),
                  c_batch=self.cb, dtype=dtype, **self.scal)
        if r.gmode != S.G_NONE:
            kw.update(mask=self.mt, strides=self.strides)
        if r.coil_mode:
            kw.update(ncoil=self.nc, coil_mode=r.coil_mode, coil_maps=self.maps)
        elif self.nc > 1:
            kw.update(ncoil=self.nc)
        return S.spectral3d_ref(c["p0"], D, H, W, **kw)

    def units(self, t):
        t = t.detach().cpu().double()
        per = self.row.coil_mode == 1 or (self.row.coil_mode == 0 and self.nc > 1)  # one unit per volume of the output
        if per:
            t = t.transpose(1, 2)
        return t.reshape(t.shape[0] * (self.nc if per else 1), -1)

    def zero_pattern_applies(self):
        r = self.row
        return r.op == FWD and r.gmode == S.G_MASK and self.binary and not r.epi


def _norms(case, got, ref):
    d = case.units(got) - case.units(ref)
    rn = case.units(ref)
    rel = d.norm(dim=1) / rn.norm(dim=1).clamp_min(1e-30)
    mx = d.abs().amax(1) / rn.abs().amax(1).clamp_min(1e-30)
    return rel, mx, float(d.norm() / rn.norm().clamp_min(1e-30))


def check_row(row: Row, dev: torch.device, emulated: bool = False) -> dict:
    from deepinv_b200 import ops

    case = Case(row, dev, row.emul if emulated and row.emul else None)
    lib = ops.get_lib()
    call = case.make_call()
    n0 = lib.dinvk_launch_count()
    got = call()
    launches = lib.dinvk_launch_count() - n0
    if dev.type == "cuda":
        torch.cuda.synchronize()
    got = got.cpu()
    assert launches == row.launches, f"{row.name}: {launches} launches, the {row.path} path issues {row.launches}"
    assert tuple(got.shape) == tuple(case.out_shape), (tuple(got.shape), case.out_shape)
    if got.numel() == 0:
        return dict(launches=launches)
    ref = case.ref(torch.float64)
    assert torch.isfinite(got).all(), row.name
    rel, mx, tot = _norms(case, got, ref)
    assert float(rel.max()) < TOL, f"{row.name}: volume {int(rel.argmax())} relative L2 error {float(rel.max()):.3g}"
    assert float(mx.max()) <= TOL, f"{row.name}: volume {int(mx.argmax())} max |error| {float(mx.max()):.3g} of max |ref|"
    res = dict(err=tot, max_rel_volume=float(rel.max()), max_abs=float(mx.max()))
    _, _, tot32 = _norms(case, case.ref(torch.float32), ref)
    res["torch32"] = tot32
    if row.path != "naive":
        assert tot <= max(4 * tot32, FLOOR), f"{row.name}: error {tot:.3g} vs torch fp32 {tot32:.3g}"
    if case.zero_pattern_applies():
        zr = ref == 0
        assert bool((got[zr] == 0).all()), f"{row.name}: nonzero k-space under the mask's zeros"
        stray = (got == 0) & ~zr
        assert bool((ref[stray].abs() <= 1e-6 * ref.abs().max()).all()), f"{row.name}: zero k-space where the mask is 1"
    if row.offset:
        al = case.make_call(0)().cpu()
        d = float((al.double() - got.double()).norm() / al.double().norm())
        assert d < 3e-6, f"{row.name}: {d:.3g} from the same call on aligned operands"
        res["vs_aligned"] = d
    return res


def einval_calls():
    """(name, kwargs of one raw `dinvk_spectral3d` call) that must return DINVK_EINVAL before touching memory"""
    big = dict(B=1, D=2048, H=1024, W=1024)
    return [("volume 2^31", big, {}),
            ("volume past 2^31", dict(B=1, D=1291, H=1291, W=1291), {}),
            ("B*D past 2^31", dict(B=1 << 20, D=4096, H=1, W=1), {}),
            ("bad D", dict(B=1, D=0, H=4, W=4), {}),
            ("stack B not a multiple of ncoil", dict(B=3, D=2, H=4, W=4), dict(ncoil=2)),
            ("coil_mode 1 adjoint", dict(B=2, D=2, H=4, W=4), dict(ncoil=2, coil_mode=1, fwd=0, inv=1)),
            ("coil_mode 2 forward", dict(B=2, D=2, H=4, W=4), dict(ncoil=2, coil_mode=2, fwd=1, inv=0)),
            ("B not a multiple of ncoil", dict(B=3, D=2, H=4, W=4), dict(ncoil=2, coil_mode=3, fwd=0, inv=1)),
            ("bad gmode", dict(B=1, D=2, H=4, W=4), dict(gmode=7))]


def run_einval(lib, dev):
    """call the raw entry with each of einval_calls(); returns [(name, rc, message)]"""
    import ctypes

    from deepinv_b200 import _ffi

    buf = torch.zeros(64, device=dev)
    out = []
    for name, shp, extra in einval_calls():
        a = _ffi.SpectralArgs()
        a.B, a.H, a.W = shp["B"], shp["H"], shp["W"]
        a.fwd, a.inv, a.centered, a.gmode = extra.get("fwd", 1), extra.get("inv", 0), 1, extra.get("gmode", 0)
        a.p0, a.out, a.a0, a.e0 = buf.data_ptr(), buf.data_ptr(), 1.0, 1.0
        a.ncoil, a.coil_mode = extra.get("ncoil", 0), extra.get("coil_mode", 0)
        a.coil_maps = buf.data_ptr()
        rc = lib.dinvk_spectral3d(ctypes.byref(a), shp["D"], ctypes.c_void_p(buf.data_ptr()), 256, None)
        out.append((name, rc, lib.dinvk_last_error()))
    return out
