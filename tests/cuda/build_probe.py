"""Build tests/cuda/libfast_arith_probe.so from fast_arith_probe.cu with the engine's own nvcc flags (no FMA contraction,
sm_90a), as a library of its own: libb200tsdf.so does not link it."""
from __future__ import annotations

import os
import subprocess

from cpu_tsdf_b200.build import CSRC, NVCC_FLAGS, _stale, nvcc_path

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "fast_arith_probe.cu")
LIB = os.path.join(HERE, "libfast_arith_probe.so")
DEPS = [SRC, __file__] + [os.path.join(CSRC, f) for f in ("obs_fast.cuh", "tsdf_core.cuh", "params_setup.h", "host_math.h")] + \
       [os.path.join(CSRC, "..", "..", "include", "b200tsdf.h"), os.path.join(CSRC, "..", "build.py")]


def build_probe(force: bool = False, out: str = LIB) -> str:
    if not force and not _stale(out, DEPS):
        return out
    ccbin = ["-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
    cmd = [nvcc_path()] + NVCC_FLAGS + ccbin + ["-shared", "-o", out, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout[-4000:] + r.stderr[-4000:])
    return out


if __name__ == "__main__":
    print(build_probe(force=True))
