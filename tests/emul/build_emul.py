"""TEST-ONLY: compile libdinvk's SIMT kernel sources for the host with g++ against cuda_emul.h.

The result (tests/emul/_build/libdinvk_emul.so) is loaded only by tests/test_emul_*.py through
ctypes with host (numpy) buffers.  The deepinv_b200 package never loads it.
"""
from __future__ import annotations

import hashlib
import subprocess
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
CSRC = ROOT / "deepinv_b200" / "csrc"
import os

# DINVK_EMUL_SANITIZE=1: AddressSanitizer + UBSan build of the emulated kernels — the CPU stand-in for compute-sanitizer's
# memcheck (out-of-bounds shared / global accesses, misaligned vector loads, signed overflow in index math).  Run with
#   DINVK_EMUL_SANITIZE=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python -m pytest tests/test_emul_kernels.py ...
SANITIZE = os.environ.get("DINVK_EMUL_SANITIZE") in ("1", "thread")
# DINVK_EMUL_SANITIZE=thread: ThreadSanitizer build — every CUDA thread is a host thread and __syncthreads / __syncwarp are real
# barriers, so a missing barrier between a shared-memory write and another thread's read is a data race TSan reports: the CPU
# stand-in for compute-sanitizer's racecheck (LD_PRELOAD=$(gcc -print-file-name=libtsan.so)).
TSAN = os.environ.get("DINVK_EMUL_SANITIZE") == "thread"
OUT = HERE / "_build" / ("libdinvk_emul_tsan.so" if TSAN else "libdinvk_emul_asan.so" if SANITIZE else "libdinvk_emul.so")
# SIMT-only translation units (the wgmma/TMA kernels cannot be emulated)
SOURCES = ["core.cu", "spectral.cu", "elementwise.cu", "radon.cu", "blur.cu", "conv_simt.cu"]
# conv_tc32.cu enters through tests/emul/conv_tc32_model.cu: its CUDA-core kernels (network head / tail, layout converters) as they
# are — the wgmma / TMA parts are compiled out — plus a test-only scalar model of the tensor-core layers behind the same C ABI
EXTRA = [HERE / "conv_tc32_model.cu"]


def build() -> Path:
    srcs = [CSRC / s for s in SOURCES if (CSRC / s).exists()] + EXTRA
    assert (CSRC / "conv_tc32.cu").exists()
    h = hashlib.sha256()
    for f in sorted(srcs + [CSRC / "conv_tc32.cu"] + list(CSRC.glob("*.cuh")) + [HERE / "cuda_emul.h", ROOT / "include" / "dinvk.h", Path(__file__)]):
        h.update(f.read_bytes())
    stamp = OUT.with_suffix(".stamp")
    if OUT.exists() and stamp.exists() and stamp.read_text() == h.hexdigest():
        return OUT
    OUT.parent.mkdir(parents=True, exist_ok=True)
    objs = []
    procs = []
    for s in srcs:
        o = OUT.parent / (s.stem + ("_tsan.o" if TSAN else "_asan.o" if SANITIZE else ".o"))
        objs.append(o)
        san = (["-fsanitize=thread", "-g", "-O1"] if TSAN else
               ["-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-g", "-O1"] if SANITIZE else ["-O2"])
        cmd = ["g++", *san, "-std=c++17", "-fPIC", "-DDINVK_EMUL", "-x", "c++", "-I", str(HERE), "-I", str(ROOT / "include"),
               "-Wno-unknown-pragmas", "-c", str(s), "-o", str(o)]
        procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise RuntimeError("emul build failed: " + " ".join(cmd))
    subprocess.run(["g++", "-shared", *(["-fsanitize=thread"] if TSAN else ["-fsanitize=address,undefined"] if SANITIZE else []), "-o", str(OUT), *map(str, objs),
                    "-lpthread"], check=True)
    stamp.write_text(h.hexdigest())
    return OUT


if __name__ == "__main__":
    print(build())
