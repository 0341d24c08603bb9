"""ctypes wrapper of the host emulation of b200tsdf_resize_pool (tests/emu/pool_emu.cpp, which compiles emu.cpp with
emu_resize_pool and raw storage accessors added).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import Config
from tests.emu import emu_py

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu_pool.so")
SRC = os.path.join(HERE, "pool_emu.cpp")


def build():
    deps = [SRC, emu_py.SRC] + [os.path.join(emu_py.CORE, f) for f in ("tsdf_core.cuh", "pool_rehash.cuh", "organize.cuh", "meshpost_core.cuh", "host_math.h", "params_setup.h")]
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in deps):
        return LIB
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++", SRC, "-o", LIB], check=True)
    return LIB


_lib = None


def load():
    global _lib
    if _lib is None:
        lib = C.CDLL(build())
        vp = C.c_void_p
        lib.emu_create.argtypes = [C.POINTER(Config)]; lib.emu_create.restype = vp
        lib.emu_destroy.argtypes = [vp]
        lib.emu_reset.argtypes = [vp]
        lib.emu_integrate.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.emu_levels.argtypes = [vp, vp]
        lib.emu_dump_nodes.argtypes = [vp] + [vp] * 6; lib.emu_dump_nodes.restype = C.c_longlong
        lib.emu_resize_pool.argtypes = [vp, C.c_int, C.c_int]
        lib.emu_pool_capacity.argtypes = [vp]; lib.emu_pool_capacity.restype = C.c_longlong
        lib.emu_pool_claimed.argtypes = [vp] + [vp] * 7; lib.emu_pool_claimed.restype = C.c_longlong
        lib.emu_unclaimed_not_fresh.argtypes = [vp]; lib.emu_unclaimed_not_fresh.restype = C.c_longlong
        lib.emu_find_keys.argtypes = [vp, vp, C.c_longlong, vp]
        lib.emu_err.argtypes = [vp]
        _lib = lib
    return _lib


class EmuPoolVolume(emu_py.EmuVolume):
    """EmuVolume over the library that also has the pool rehash"""

    def __init__(self, **kw):
        lib = load()
        saved = emu_py._lib
        emu_py._lib = lib                      # EmuVolume.__init__ binds the library it loads
        try:
            super().__init__(**kw)
        finally:
            emu_py._lib = saved

    def resize_pool(self, pool_log2: int, check_fit: bool = True) -> int:
        """0 installed, 1 over the load limit, 2 a brick hit MAX_PROBE, 3 pool_log2 out of range"""
        return self.lib.emu_resize_pool(self.h, int(pool_log2), int(check_fit))

    def err(self) -> int:
        return self.lib.emu_err(self.h)

    def capacity(self) -> int:
        return self.lib.emu_pool_capacity(self.h)

    def claimed(self):
        """the claimed slots in slot order: slot numbers, keys, {d, w} nodes, split words, and rgb / M / ns when the volume
        has them"""
        n = self.lib.emu_pool_claimed(self.h, *([None] * 7))
        out = {"slots": np.empty(n, np.int32), "keys": np.empty(n, np.uint64), "nodes": np.empty((n, 584, 2), np.float32),
               "split": np.empty((n, 20), np.uint32)}
        if self.cfg.integrate_color:
            out["rgb"] = np.empty((n, 584, 4), np.uint8)
        if self.cfg.track_variance:
            out["M"] = np.empty((n, 584), np.float32); out["ns"] = np.empty((n, 584), np.int32)
        p = emu_py._ptr
        self.lib.emu_pool_claimed(self.h, p(out["slots"]), p(out["keys"]), p(out["nodes"]), p(out["split"]), p(out.get("rgb")),
                                  p(out.get("M")), p(out.get("ns")))
        return out

    def unclaimed_not_fresh(self) -> int:
        return self.lib.emu_unclaimed_not_fresh(self.h)

    def find(self, keys) -> np.ndarray:
        keys = np.ascontiguousarray(keys, np.uint64)
        out = np.empty(len(keys), np.int32)
        self.lib.emu_find_keys(self.h, emu_py._ptr(keys), len(keys), emu_py._ptr(out))
        return out
