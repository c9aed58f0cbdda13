"""Build libdinvk.so (the sm_90a kernel library) in-tree with nvcc.

The shared object is a build product (git-ignored).
`python -m deepinv_b200.build` rebuilds it; `__graft_entry__.build()` calls `build()`.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
LIB = PKG / "libdinvk.so"
STAMP = PKG / ".libdinvk.stamp"

NVCC_FLAGS = [
    "-O3",
    "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--use_fast_math=false",
    "-Xcompiler", "-fPIC",
    "-shared",
]


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [ROOT / "include" / "dinvk.h", Path(__file__)]):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    dig = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    tmp = LIB.with_suffix(".so.tmp")  # link to a scratch name, then rename: a reader never sees a half-written library
    cmd = [nvcc, *flags, "-I", str(ROOT / "include"), "-o", str(tmp), *map(str, sources())]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True, cwd=str(ROOT))
    os.replace(tmp, LIB)
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
