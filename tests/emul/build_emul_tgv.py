"""TEST-ONLY: compile the TGV kernels (deepinv_b200/csrc/tv.cu) for the host with g++ against cuda_emul.h.

Like build_emul_tv.py (core.cu + tv.cu, the same flags and sanitizer modes), but `build(tile, block)` can override the
compile-time tile edge DINVK_TGV_TILE and iterations per launch DINVK_TGV_BLOCK, so that tests can check that the
choice changes no output bit.  Each (tile, block) pair gets a library of its own under tests/emul/_build/.
"""
from __future__ import annotations

import hashlib
import subprocess
from pathlib import Path

from build_emul import CSRC, HERE, ROOT, SANITIZE, TSAN

SOURCES = ["core.cu", "tv.cu"]


def build(tile: int | None = None, block: int | None = None) -> Path:
    defs = ([f"-DDINVK_TGV_TILE={tile}"] if tile else []) + ([f"-DDINVK_TGV_BLOCK={block}"] if block else [])
    tag = "".join(f"_{v}" for v in (tile, block) if v) + ("_tsan" if TSAN else "_asan" if SANITIZE else "")
    out = HERE / "_build" / f"libdinvk_emul_tgv{tag}.so"
    srcs = [CSRC / s for s in SOURCES]
    h = hashlib.sha256(" ".join(defs).encode())
    for f in sorted(srcs + list(CSRC.glob("*.cuh")) + [HERE / "cuda_emul.h", ROOT / "include" / "dinvk.h", Path(__file__)]):
        h.update(f.read_bytes())
    stamp = out.with_suffix(".stamp")
    if out.exists() and stamp.exists() and stamp.read_text() == h.hexdigest():
        return out
    out.parent.mkdir(parents=True, exist_ok=True)
    san = (["-fsanitize=thread", "-g", "-O1"] if TSAN else
           ["-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-g", "-O1"] if SANITIZE else ["-O2"])
    objs, procs = [], []
    for s in srcs:
        o = out.parent / (f"tgvlib{tag}_" + s.stem + ".o")
        objs.append(o)
        cmd = ["g++", *san, *defs, "-std=c++17", "-fPIC", "-DDINVK_EMUL", "-x", "c++", "-I", str(HERE), "-I", str(ROOT / "include"),
               "-Wno-unknown-pragmas", "-c", str(s), "-o", str(o)]
        procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise RuntimeError("emul build failed: " + " ".join(cmd))
    subprocess.run(["g++", "-shared", *(["-fsanitize=thread"] if TSAN else ["-fsanitize=address,undefined"] if SANITIZE else []),
                    "-o", str(out), *map(str, objs), "-lpthread"], check=True)
    stamp.write_text(h.hexdigest())
    return out


if __name__ == "__main__":
    print(build())
