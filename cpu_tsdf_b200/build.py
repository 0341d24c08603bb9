"""In-tree build of libb200tsdf.so for sm_90a (H100; nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200tsdf.so")
# source -> headers it includes (csrc/), for incremental rebuilds
SOURCES = {
    "engine.cu": ["tsdf_core.cuh", "mc_tables.cuh", "host_math.h", "params_setup.h", "brick_kernels.cuh", "obs_fast.cuh", "brick_direct.cuh", "multigpu.cuh", "organize.cuh", "mesh_sort.h", "host_pack.h"],
    "meshpost.cu": ["tsdf_core.cuh", "meshpost_core.cuh", "mesh_sort.h"],
}
OBJ = os.path.join(CSRC, "_obj")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # every float expression must round exactly as the reference's: no FMA contraction anywhere
    "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off,-O2",
    "-Xptxas", "-v",
]


def nvcc_path() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _deps(src: str) -> list[str]:
    return [os.path.join(CSRC, f) for f in [src] + SOURCES[src]] + [os.path.join(HERE, "..", "include", "b200tsdf.h"), __file__]


def needs_build() -> bool:
    return any(_stale(LIB, _deps(s)) for s in SOURCES)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """nvcc -c per source (only the stale ones, in parallel), then one link into libb200tsdf.so."""
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    ccbin = ["-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
    jobs = []
    for src in SOURCES:
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(obj, _deps(src)):
            cmd = [nvcc_path()] + NVCC_FLAGS + ccbin + ["-c", "-o", obj, os.path.join(CSRC, src)]
            jobs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    out = ""
    failed = False
    for cmd, pr in jobs:
        o, _ = pr.communicate()
        out += " ".join(cmd) + "\n" + o
        failed |= pr.returncode != 0
    if not failed:
        cmd = [nvcc_path(), "-shared"] + ccbin + ["-o", LIB] + [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
        r = subprocess.run(cmd, capture_output=True, text=True)
        out += " ".join(cmd) + "\n" + r.stdout + r.stderr
        failed = r.returncode != 0
    # keep the ptxas -v output of every object in the log, also of those that were not recompiled this time
    log = os.path.join(HERE, "build.log")
    with open(log, "w" if force or len(jobs) == len(SOURCES) else "a") as f:
        f.write(out)
    if verbose:
        print(out)
    if failed:
        raise RuntimeError("nvcc failed:\n" + out[-8000:])
    return LIB


# ---- host programs above the C ABI (the reference's src/prog equivalents) ---------------------------------------
PROG = os.path.join(HERE, "prog")
BIN = os.path.join(HERE, "bin")
PROGRAMS = {                       # name -> needs libb200tsdf
    "b200_integrate": True, "b200_tsdf2mesh": True, "b200_pcd_convert": False,
}


def build_programs(force: bool = False) -> list[str]:
    """g++ the programs under prog/ into bin/ (rpath $ORIGIN/.. so they find libb200tsdf.so in-tree)."""
    os.makedirs(BIN, exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    inc = os.path.join(HERE, "..", "include")
    hdrs = [os.path.join(PROG, f) for f in os.listdir(PROG) if f.endswith(".h")] + \
           [os.path.join(inc, "b200tsdf.h"), os.path.join(inc, "cpu_tsdf_b200", "tsdf_volume_octree.h"), os.path.join(CSRC, "host_math.h")]
    out = []
    for name, needs_lib in PROGRAMS.items():
        src, exe = os.path.join(PROG, name + ".cpp"), os.path.join(BIN, name)
        if force or _stale(exe, [src] + hdrs + ([LIB] if needs_lib else [])):
            cmd = [cxx, "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-I" + inc, src, "-o", exe]
            if needs_lib:
                cmd += ["-L" + HERE, "-lb200tsdf", "-Wl,-rpath,$ORIGIN/.."]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
        out.append(exe)
    return out
