"""TEST-ONLY: compile the TV kernels (deepinv_b200/csrc/tv.cu) for the host with g++ against cuda_emul.h.

A library of its own (tests/emul/_build/libdinvk_emul_tv*.so, core.cu + tv.cu), built with the same flags and sanitizer
modes (DINVK_EMUL_SANITIZE=1 / =thread) as build_emul.py, and loaded only by tests/test_emul_tv.py through ctypes.
"""
from __future__ import annotations

import hashlib
import subprocess
from pathlib import Path

from build_emul import CSRC, HERE, ROOT, SANITIZE, TSAN

OUT = HERE / "_build" / ("libdinvk_emul_tv_tsan.so" if TSAN else "libdinvk_emul_tv_asan.so" if SANITIZE else "libdinvk_emul_tv.so")
SOURCES = ["core.cu", "tv.cu"]


def build() -> Path:
    srcs = [CSRC / s for s in SOURCES]
    h = hashlib.sha256()
    for f in sorted(srcs + list(CSRC.glob("*.cuh")) + [HERE / "cuda_emul.h", ROOT / "include" / "dinvk.h", Path(__file__)]):
        h.update(f.read_bytes())
    stamp = OUT.with_suffix(".stamp")
    if OUT.exists() and stamp.exists() and stamp.read_text() == h.hexdigest():
        return OUT
    OUT.parent.mkdir(parents=True, exist_ok=True)
    san = (["-fsanitize=thread", "-g", "-O1"] if TSAN else
           ["-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-g", "-O1"] if SANITIZE else ["-O2"])
    objs, procs = [], []
    for s in srcs:
        o = OUT.parent / ("tvlib_" + s.stem + ("_tsan.o" if TSAN else "_asan.o" if SANITIZE else ".o"))
        objs.append(o)
        cmd = ["g++", *san, "-std=c++17", "-fPIC", "-DDINVK_EMUL", "-x", "c++", "-I", str(HERE), "-I", str(ROOT / "include"),
               "-Wno-unknown-pragmas", "-c", str(s), "-o", str(o)]
        procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise RuntimeError("emul build failed: " + " ".join(cmd))
    subprocess.run(["g++", "-shared", *(["-fsanitize=thread"] if TSAN else ["-fsanitize=address,undefined"] if SANITIZE else []),
                    "-o", str(OUT), *map(str, objs), "-lpthread"], check=True)
    stamp.write_text(h.hexdigest())
    return OUT


if __name__ == "__main__":
    print(build())
