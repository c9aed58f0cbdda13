"""One case table for every launch path of `dinvk_spectral`, shared by the H100 run (tests/test_gpu_spectral_paths.py) and the
host-emulated twin (tests/test_emul_spectral_paths.py).

The host code picks a kernel family from the image size, the operation and pointer alignment (csrc/spectral.cu): the pipelined
256² / 320² kernels, the power-of-two fast tile kernels (N = 64 .. 1024), the generic mixed-radix tile passes at 256 / 512 / 1024
threads with 16-, 8- or 4-column strips, the O(N²) axis DFT for sizes with a prime factor above 5 or beyond the tile budget, the
elementwise-only pass, and the coil reduction after any of them.  Each row names the family it is meant to reach and the number
of launches that family issues; the launch count pins the branch, the kernel census of the GPU file pins the kernels.

Every row is checked against the fp64 contract (tests/spectral_ref64.py), or for the BlurFFT rows against oracle/ref_ops.py in
float64:
  * relative L2 error per image (per image and coil for coil_mode 1) < 1e-5;
  * max |error| per image <= 1e-5 * max |ref| of that image (a wrong strip, tile or image is not diluted by the batch);
  * off the O(N²) path: error <= max(4 x the error of torch's own fp32 evaluation of the same contract, 5e-7);
  * the exact zero pattern of a 0/1-masked `A` (a sample under a mask 1 may round to 0 only if its true value is
    below 1e-6 of the largest: fp32 cancellation, seen once in 13 M samples of the 16-coil brain rows);
  * rows whose operands sit off 16-byte alignment also agree within 3e-6 with the same call on aligned copies.
"""
from __future__ import annotations

import dataclasses
import zlib
from typing import Optional

import torch

import spectral_ref64 as S

TOL = 1e-5
FLOOR = 5e-7

FWD, ADJ, FUSED, ELEM = (1, 0), (0, 1), (1, 1), (0, 0)


@dataclasses.dataclass(frozen=True)
class Row:
    name: str
    shape: tuple            # (B, H, W); B counts batch samples (coil images are B * ncoil)
    op: tuple               # (fwd, inv)
    gmode: int
    mask: str               # none | line | full | shared | weighted | cplx | cplx_line
    path: str               # pipe | fast | tile | naive | elem (the family the row is meant to reach)
    launches: int
    centered: bool = True
    epi: bool = False       # a0, p1 / a1, e0, q0 / e1, q1 / e2 all present
    prox: bool = False      # p1 with a1 = c = 1 / gamma (prox_l2)
    cb: bool = False        # per-image constants c_batch
    ncoil: int = 0
    coil_mode: int = 0
    maps: str = "shared"    # shared | per (coil maps (1|B, ncoil, H, W))
    e0: float = 1.0
    offset: int = 0         # p0, p1, q0 and the multiplier start `offset` floats into their allocation
    blur: str = ""          # BlurFFT method (A, At, prox, dagger) of a physics-class row
    channels: int = 1
    filt: str = "shared"    # shared | per (one filter per sample and channel)
    emul: Optional[tuple] = None  # smaller (B, H, W) for the host emulation, on the same path with the same launch count


def _row(name, shape, op, gmode, mask, path, launches, **kw):
    return Row(name, shape, op, gmode, mask, path, launches, **kw)


def _rows():
    R = []
    # ---- FastMRI knee, single coil: 640 x 368 (16 * 23) and 640 x 372 (4 * 3 * 31) go down the O(N²) path ---------------------
    for W, em in ((368, (2, 40, 46)), (372, (1, 24, 62))):
        k = f"knee{W}"
        for m in ("line", "full"):
            R += [_row(f"{k} A {m}", (2, 640, W), FWD, S.G_MASK, m, "naive", 4, emul=em),
                  _row(f"{k} At {m}", (2, 640, W), ADJ, S.G_MASK, m, "naive", 4, emul=em),
                  _row(f"{k} AtA {m}", (2, 640, W), FUSED, S.G_SQ, m, "naive", 7, emul=em),
                  _row(f"{k} prox {m}", (2, 640, W), FUSED, S.G_INV_SQ_PLUS_C, m, "naive", 7, prox=True, emul=em)]
        R += [_row(f"{k} dagger line", (2, 640, W), ADJ, S.G_PINV, "line", "naive", 4, emul=em),
              _row(f"{k} dagger weighted", (2, 640, W), ADJ, S.G_PINV, "weighted", "naive", 4, emul=em)]
    # ---- FastMRI knee, 15 coils: O(N²) transforms, then the coil reduction fed by the cudaMemcpyAsync branch ------------------
    for mode in (1, 2, 3):
        R.append(_row(f"knee368 15 coils mode {mode}", (1, 640, 368), FWD if mode == 1 else ADJ, S.G_MASK, "line", "naive", 4,
                      ncoil=15, coil_mode=mode, e0=0.7 if mode == 2 else 1.0, emul=(1, 40, 46)))
    # ---- FastMRI brain, 16 coils, 640 x 320: generic column pass at 1024 threads ---------------------------------------------
    for maps in ("shared", "per"):
        for mode in (1, 2, 3):
            R.append(_row(f"brain 16 coils {maps} maps mode {mode}", (2, 640, 320), FWD if mode == 1 else ADJ, S.G_MASK, "line",
                          "tile", 2 if mode == 1 else 3, ncoil=16, coil_mode=mode, maps=maps, e0=0.7 if mode == 2 else 1.0,
                          emul=(2, 640, 20)))
    # ---- column strips: 8 columns (H in (960, 1920]), 4 columns, and past the tile budget -------------------------------------
    for H, W in ((1080, 40), (1200, 40), (2000, 8)):
        R += [_row(f"strips {H}x{W} A", (2, H, W), FWD, S.G_MASK, "full", "tile", 2),
              _row(f"strips {H}x{W} At", (2, H, W), ADJ, S.G_MASK, "full", "tile", 2),
              _row(f"strips {H}x{W} AtA", (2, H, W), FUSED, S.G_SQ, "full", "tile", 3)]
    R += [_row("5000x4 A", (1, 5000, 4), FWD, S.G_MASK, "full", "naive", 4),
          _row("5000x4 At", (1, 5000, 4), ADJ, S.G_MASK, "full", "naive", 4),
          _row("5000x4 AtA", (1, 5000, 4), FUSED, S.G_SQ, "full", "naive", 7)]
    # ---- wide rows: row pass at 512 (W = 4800) and 1024 threads (W = 9600) ----------------------------------------------------
    for W in (4800, 9600):
        H = 4 if W == 4800 else 2
        em = (1, H, W)
        R += [_row(f"wide {H}x{W} A", (2, H, W), FWD, S.G_MASK, "full", "tile", 2, emul=em),
              _row(f"wide {H}x{W} At", (2, H, W), ADJ, S.G_MASK, "full", "tile", 2, emul=em),
              _row(f"wide {H}x{W} AtA line", (2, H, W), FUSED, S.G_SQ, "line", "tile", 1, emul=em),
              _row(f"wide {H}x{W} AtA full", (2, H, W), FUSED, S.G_SQ, "full", "tile", 3, emul=em)]
    # ---- the 15-element budget of a radix-3/5 plan: 16 * threads would fit these tiles, 15 * threads does not -----------------
    R += [_row("budget 1000x40 A", (2, 1000, 40), FWD, S.G_MASK, "full", "tile", 2),
          _row("budget 1000x40 At", (2, 1000, 40), ADJ, S.G_MASK, "full", "tile", 2),
          _row("budget 2x4000 A", (2, 2, 4000), FWD, S.G_MASK, "full", "tile", 2),
          _row("budget 2x4000 At", (2, 2, 4000), ADJ, S.G_MASK, "full", "tile", 2),
          _row("budget 2x4000 AtA line", (2, 2, 4000), FUSED, S.G_SQ, "line", "tile", 1)]
    # ---- fast kernels: 512 both ways, the 128 row kernel next to a generic column pass, 1024 --------------------------------
    R += [_row("fast 512 A", (2, 512, 512), FWD, S.G_MASK, "full", "fast", 2),
          _row("fast 512 At", (2, 512, 512), ADJ, S.G_MASK, "full", "fast", 2),
          _row("fast 512 AtA full", (2, 512, 512), FUSED, S.G_SQ, "full", "fast", 3, emul=(1, 512, 512)),
          _row("fast 512 prox full", (2, 512, 512), FUSED, S.G_INV_SQ_PLUS_C, "full", "fast", 3, prox=True),
          _row("fast 96x128 A", (4, 96, 128), FWD, S.G_MASK, "full", "fast", 2),
          _row("fast 96x128 At", (4, 96, 128), ADJ, S.G_MASK, "full", "fast", 2),
          _row("fast 1024 AtA full", (1, 1024, 1024), FUSED, S.G_SQ, "full", "fast", 3, emul=(1, 1024, 64))]
    # ---- fast-path fallbacks on geometry: H % 8 != 0 (row pass generic), W % 16 != 0 (column pass generic, short last strip) --
    R += [_row("geom 100x512 A", (3, 100, 512), FWD, S.G_MASK, "full", "tile", 2),
          _row("geom 100x512 At", (3, 100, 512), ADJ, S.G_MASK, "full", "tile", 2),
          _row("geom 256x200 A", (2, 256, 200), FWD, S.G_MASK, "full", "tile", 2),
          _row("geom 256x200 At", (2, 256, 200), ADJ, S.G_MASK, "full", "tile", 2),
          _row("geom 256x200 AtA full", (2, 256, 200), FUSED, S.G_SQ, "full", "tile", 3)]
    # ---- odd smooth size 405 x 243 (3^4 * 5 x 3^5): centred and plain transforms differ at odd N ------------------------------
    for cen in (True, False):
        c = "centred" if cen else "plain"
        R += [_row(f"odd 405x243 A {c}", (2, 405, 243), FWD, S.G_MASK, "full", "tile", 2, centered=cen),
              _row(f"odd 405x243 At {c}", (2, 405, 243), ADJ, S.G_MASK, "full", "tile", 2, centered=cen),
              _row(f"odd 405x243 AtA {c}", (2, 405, 243), FUSED, S.G_SQ, "full", "tile", 3, centered=cen)]
    # ---- alignment fallbacks: operands 4 or 8 bytes off 16-byte alignment leave the pipelined and fast kernels ----------------
    for N in (256, 320):
        for off in (1, 2):
            a = f"align {N} +{off}"
            R += [_row(f"{a} A full", (2, N, N), FWD, S.G_MASK, "full", "tile", 2, epi=True, offset=off),
                  _row(f"{a} At line", (2, N, N), ADJ, S.G_MASK, "line", "tile", 2, epi=True, offset=off),
                  _row(f"{a} AtA line", (2, N, N), FUSED, S.G_SQ, "line", "tile", 1, epi=True, offset=off),
                  _row(f"{a} AtA full", (2, N, N), FUSED, S.G_SQ, "full", "tile", 3, epi=True, offset=off, emul=(1, N, N))]
    # ---- every gmode, c_batch and the full epilogue, once per family: O(N²) (odd sizes), generic at 1024 threads, fast at 512 --
    fams = (("naive", (2, 117, 93), 4, 7, 7, None), ("tile", (2, 640, 320), 2, 3, 1, (1, 640, 40)),
            ("fast", (2, 512, 512), 2, 3, 1, (1, 512, 512)))
    for fam, shape, n1, n3, nline, em in fams:
        f = f"gmodes {fam} {shape[1]}x{shape[2]}"
        for gm, m in ((S.G_MASK, "full"), (S.G_SQ, "weighted"), (S.G_INV_SQ_PLUS_C, "weighted"), (S.G_PINV, "weighted"),
                      (S.G_CMUL, "cplx"), (S.G_CMUL_CONJ, "cplx")):
            R.append(_row(f"{f} fused g{gm}", shape, FUSED, gm, m, fam, n3, epi=True, centered=gm < S.G_CMUL, emul=em))
        R += [_row(f"{f} A g1", shape, FWD, S.G_MASK, "full", fam, n1, epi=True, emul=em),
              _row(f"{f} At g4", shape, ADJ, S.G_PINV, "weighted", fam, n1, epi=True, emul=em),
              _row(f"{f} fused g3 c_batch", shape, FUSED, S.G_INV_SQ_PLUS_C, "weighted", fam, n3, cb=True, prox=True, emul=em),
              _row(f"{f} fused g5 line", shape, FUSED, S.G_CMUL, "cplx_line", fam, nline, centered=False, emul=em)]
    # ---- elementwise only (fwd = inv = 0), every gmode, at a size that is not a power of two -----------------------------------
    for gm, m in ((S.G_NONE, "none"), (S.G_MASK, "full"), (S.G_SQ, "weighted"), (S.G_INV_SQ_PLUS_C, "weighted"),
                  (S.G_PINV, "weighted"), (S.G_CMUL, "cplx"), (S.G_CMUL_CONJ, "cplx")):
        R.append(_row(f"elementwise g{gm}", (3, 90, 70), ELEM, gm, m, "elem", 1, epi=True))
    R.append(_row("elementwise g3 c_batch", (3, 90, 70), ELEM, S.G_INV_SQ_PLUS_C, "weighted", "elem", 1, cb=True))
    # ---- BlurFFT through the physics class: 1080p, C = 3 (odd B * C: the zero-padded pair), 31 x 31 filter; 720p per-image ----
    for meth, n in (("A", 3), ("At", 3), ("prox", 6), ("dagger", 3)):
        R.append(_row(f"blurfft 1080x1920 C3 {meth}", (1, 1080, 1920), FUSED, S.G_CMUL, "cplx", "tile", n, blur=meth, channels=3,
                      emul=(1, 60, 80)))
        R.append(_row(f"blurfft 720x1280 per-image {meth}", (2, 720, 1280), FUSED, S.G_CMUL, "cplx", "tile", n, blur=meth,
                      channels=3, filt="per", emul=(2, 40, 48)))
    names = [r.name for r in R]
    assert len(names) == len(set(names))
    return R


ROWS = _rows()


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------
def _mask(kind, B, H, W, g):
    """(tensor, (sb, sc, sh), complex?, binary?) in the ABI's addressing (dinvk.h)"""
    if kind == "line":
        t = (torch.rand(B, 1, 1, W, generator=g) > 0.4).float()
        return t, (W if B > 1 else 0, 0, 0), False, True
    if kind == "full":
        return (torch.rand(B, 2, H, W, generator=g) > 0.5).float(), (2 * H * W, H * W, W), False, True
    if kind == "shared":
        return (torch.rand(1, 2, H, W, generator=g) > 0.5).float(), (0, H * W, W), False, True
    if kind == "weighted":  # zeros, values below the pseudo-inverse threshold, and weights in (0.05, 1)
        t = (0.05 + 0.95 * torch.rand(B, 2, H, W, generator=g)) * (torch.rand(B, 2, H, W, generator=g) > 0.3).float()
        t.view(-1)[::97] = 3e-6
        return t, (2 * H * W, H * W, W), False, False
    if kind == "cplx":
        return torch.randn(B, H, W, 2, generator=g), (H * W, 0, W), True, False
    if kind == "cplx_line":
        return torch.randn(B, 1, W, 2, generator=g), (W if B > 1 else 0, 0, 0), True, False
    raise ValueError(kind)


class Case:
    """the inputs of one row on one device, the call, and its references"""

    def __init__(self, row: Row, dev: torch.device, shape=None):
        self.row, self.dev = row, dev
        B, H, W = self.shape = tuple(shape or row.shape)
        self.g = torch.Generator().manual_seed(zlib.crc32(row.name.encode()))
        if row.blur:
            self._init_blur()
            self._blur_fn = self._blur_call()  # the physics object and its multipliers are built outside the counted call
            return
        g = self.g
        nc = row.ncoil if row.ncoil > 1 else 1
        self.nc = nc
        src = (B, 2, nc, H, W) if nc > 1 and row.coil_mode >= 2 else (B, 2, H, W)
        self.out_shape = {1: (B, 2, nc, H, W), 2: (B, 2, H, W), 3: (B, 1, H, W)}.get(row.coil_mode if nc > 1 else 0, (B, 2, H, W))
        c = {}
        c["p0"] = torch.randn(src, generator=g)
        if row.epi or row.prox:
            c["p1"] = torch.randn(src, generator=g)
        if row.epi:
            c["q0"] = torch.randn(self.out_shape, generator=g)
            c["q1"] = torch.randn(self.out_shape, generator=g)
        self.cpu = c
        self.binary = False
        if row.gmode != S.G_NONE:
            self.mt, self.strides, self.cplx, self.binary = _mask(row.mask, B, H, W, g)
        self.scal = dict(a0=0.5 if row.epi else 1.0, a1=-1.5 if row.epi else (1 / 0.7 if row.prox else 0.0),
                         e0=2.0 if row.epi else row.e0, e1=0.25 if row.epi else 0.0, e2=-0.75 if row.epi else 0.0, c=1 / 0.7)
        self.cb = (torch.rand(B, generator=g) + 0.5) if row.cb else None
        self.maps = None
        if nc > 1:
            mp = torch.randn(1 if row.maps == "shared" else B, nc, H, W, generator=g, dtype=torch.complex64)
            self.maps = (mp / mp.abs().pow(2).sum(1, keepdim=True).sqrt()).contiguous()

    # ---- spectral rows ------------------------------------------------------------------------------------------------------
    def _place(self, t, offset):
        if offset == 0:
            return t.to(self.dev).contiguous()
        flat = torch.zeros(t.numel() + offset, dtype=t.dtype, device=self.dev)
        flat[offset:] = t.reshape(-1).to(self.dev)
        return flat[offset:].view(t.shape)

    def _call(self, offset):
        from deepinv_b200 import ops

        r = self.row
        B, H, W = self.shape
        d = {k: self._place(v, offset if k != "q1" else 0) for k, v in self.cpu.items()}
        kw = dict(fwd=bool(r.op[0]), inv=bool(r.op[1]), centered=r.centered, gmode=r.gmode, c=self.scal["c"],
                  a0=self.scal["a0"], a1=self.scal["a1"], e0=self.scal["e0"], e1=self.scal["e1"], e2=self.scal["e2"],
                  p1=d.get("p1"), q0=d.get("q0"), q1=d.get("q1"))
        if r.gmode != S.G_NONE:
            sb, sc, sh = self.strides
            kw["mask"] = ops.MaskSpec(self._place(self.mt, offset), sb, sc, sh, self.cplx)
        if self.cb is not None:
            kw["c_batch"] = self.cb.to(self.dev)
        if self.nc > 1:
            kw.update(ncoil=self.nc, coil_mode=r.coil_mode, coil_maps=self.maps.to(self.dev))
        return lambda: ops.spectral(d["p0"], H, W, **kw)

    def run(self):
        """the call under test (at the row's offset)"""
        return self._blur_fn() if self.row.blur else self._call(self.row.offset)()

    def run_aligned(self):
        return self._call(0)()

    def ref(self, dtype=torch.float64):
        if self.row.blur:
            return self._blur_ref(dtype)
        r = self.row
        B, H, W = self.shape
        c = self.cpu
        kw = dict(fwd=r.op[0], inv=r.op[1], centered=r.centered, gmode=r.gmode, p1=c.get("p1"), q0=c.get("q0"), q1=c.get("q1"),
                  c_batch=self.cb, dtype=dtype, **self.scal)
        if r.gmode != S.G_NONE:
            kw.update(mask=self.mt, strides=self.strides)
        if self.nc > 1:
            kw.update(ncoil=self.nc, coil_mode=r.coil_mode, coil_maps=self.maps)
        return S.spectral_ref(c["p0"], H, W, **kw)

    def units(self, t):
        """(images, elements): one row per image (per image and coil for coil_mode 1)"""
        t = t.detach().cpu().double()
        if self.row.blur:
            return t.reshape(-1, self.shape[1] * self.shape[2])
        if self.nc > 1 and self.row.coil_mode == 1:
            t = t.transpose(1, 2)
        return t.reshape(t.shape[0] * (self.nc if self.nc > 1 and self.row.coil_mode == 1 else 1), -1)

    def zero_pattern_applies(self):
        r = self.row
        return (not r.blur and r.op == FWD and r.gmode == S.G_MASK and self.binary and not r.epi)

    # ---- BlurFFT rows ---------------------------------------------------------------------------------------------------------
    def _init_blur(self):
        r, g = self.row, self.g
        B, H, W = self.shape
        C = r.channels
        fb, fc = (B, C) if r.filt == "per" else (1, 1)
        k = min(31, H // 2 * 2 - 1, W // 2 * 2 - 1)
        f = torch.rand(fb, fc, k, k, generator=g)
        f = 0.4 * f / f.sum((-2, -1), keepdim=True)
        f[..., k // 2, k // 2] += 0.6  # |spectrum| >= 0.2: the pseudo-inverse stays well conditioned
        self.filt = f
        self.x = torch.randn(B, C, H, W, generator=g)
        self.z = torch.randn(B, C, H, W, generator=g)
        self.gamma = 0.7

    def _blur_call(self):
        import deepinv_b200 as dinv

        B, H, W = self.shape
        C = self.row.channels
        phys = dinv.physics.BlurFFT(img_size=(C, H, W), filter=self.filt.to(self.dev), device=self.dev)
        phys._mult()
        x, z = self.x.to(self.dev), self.z.to(self.dev)
        m = self.row.blur

        def call():
            with torch.no_grad():
                if m == "A":
                    return phys.A(x)
                if m == "At":
                    return phys.A_adjoint(x)
                if m == "prox":
                    return phys.prox_l2(z, x, self.gamma)
                return phys.A_dagger(x)
        return call

    def _blur_ref(self, dtype):
        from oracle import ref_ops as R

        B, H, W = self.shape
        img = (self.row.channels, H, W)
        mask, angle = R.blurfft_params(self.filt.to(dtype), img)
        x, z = self.x.to(dtype), self.z.to(dtype)
        m = self.row.blur
        if m == "A":
            return R.blurfft_A(x, mask, angle, img)
        if m == "At":
            return R.blurfft_At(x, mask, angle, img)
        if m == "prox":
            return R.blurfft_prox_l2(z, x, mask, angle, img, self.gamma)
        return R.blurfft_dagger(x, mask, angle, img)


def _norms(case, got, ref):
    d = case.units(got) - case.units(ref)
    rn = case.units(ref)
    rel = d.norm(dim=1) / rn.norm(dim=1).clamp_min(1e-30)
    mx = d.abs().amax(1) / rn.abs().amax(1).clamp_min(1e-30)
    return rel, mx, float(d.norm() / rn.norm().clamp_min(1e-30))


def check_row(row: Row, dev: torch.device, emulated: bool = False) -> dict:
    """run one row, assert every property of the module docstring, return the measured errors"""
    from deepinv_b200 import ops

    case = Case(row, dev, row.emul if emulated and row.emul else None)
    lib = ops.get_lib()
    n0 = lib.dinvk_launch_count()
    got = case.run()
    launches = lib.dinvk_launch_count() - n0
    if dev.type == "cuda":
        torch.cuda.synchronize()
    got = got.cpu()
    assert launches == row.launches, f"{row.name}: {launches} launches, the {row.path} path issues {row.launches}"
    ref = case.ref(torch.float64)
    assert tuple(got.shape) == tuple(ref.shape), (tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all(), row.name
    rel, mx, tot = _norms(case, got, ref)
    worst = int(rel.argmax())
    assert float(rel.max()) < TOL, f"{row.name}: image {worst} relative L2 error {float(rel.max()):.3g}"
    assert float(mx.max()) <= TOL, f"{row.name}: image {int(mx.argmax())} max |error| {float(mx.max()):.3g} of max |ref|"
    res = dict(err=tot, max_rel_image=float(rel.max()), max_abs=float(mx.max()))
    _, _, tot32 = _norms(case, case.ref(torch.float32), ref)
    res["torch32"] = tot32
    if row.path != "naive":  # the O(N²) path sums N products per output: held to TOL only, its error is reported
        assert tot <= max(4 * tot32, FLOOR), f"{row.name}: error {tot:.3g} vs torch fp32 {tot32:.3g}"
    if case.zero_pattern_applies():
        # exact zeros wherever the mask is 0; elsewhere an exact 0 only where the true value is below fp32 cancellation level
        zr = ref == 0
        assert bool((got[zr] == 0).all()), f"{row.name}: nonzero k-space under the mask's zeros"
        stray = (got == 0) & ~zr
        assert bool((ref[stray].abs() <= 1e-6 * ref.abs().max()).all()), f"{row.name}: zero k-space where the mask is 1"
    if row.offset:
        al = case.run_aligned().cpu()
        d = float((al.double() - got.double()).norm() / al.double().norm())
        assert d < 3e-6, f"{row.name}: {d:.3g} from the same call on aligned operands"
        res["vs_aligned"] = d
    return res
