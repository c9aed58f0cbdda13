"""TEST-ONLY: compile the TV and TGV kernels (deepinv_b200/csrc/tv.cu) for the host with g++ against cuda_emul.h.

A library of its own per set of -D overrides (tests/emul/_build/libdinvk_emul_tv*.so, core.cu + tv.cu), such as
`build(DINVK_TGV_TILE=20, DINVK_TGV_BLOCK=3)`, so that tests can check that T and K change no output bit; the same flags
and sanitizer modes (DINVK_EMUL_SANITIZE=1 / =thread) as build_emul.py.
"""
from __future__ import annotations

import hashlib
import subprocess
from pathlib import Path

from build_emul import CSRC, HERE, ROOT, SANITIZE, TSAN

SOURCES = ["core.cu", "tv.cu"]


def build(**defines: int) -> Path:
    defs = [f"-D{k}={int(v)}" for k, v in sorted(defines.items())]
    tag = "".join(f"_{k[6:].lower()}{int(v)}" for k, v in sorted(defines.items())) + ("_tsan" if TSAN else "_asan" if SANITIZE else "")
    out = HERE / "_build" / f"libdinvk_emul_tv{tag}.so"
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
        o = out.parent / (f"tvlib{tag}_" + s.stem + ".o")
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
