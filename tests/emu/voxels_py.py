"""ctypes wrapper of the host emulation of the point lookup and the dense crop (tests/emu/voxels_emu.cpp, which compiles
emu.cpp with emu_voxels / emu_dense added).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import VOXEL_DTYPE, Config
from tests.emu import emu_py

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu_voxels.so")
SRC = os.path.join(HERE, "voxels_emu.cpp")


def build():
    deps = [SRC, emu_py.SRC] + [os.path.join(emu_py.CORE, f) for f in ("tsdf_core.cuh", "organize.cuh", "meshpost_core.cuh", "host_math.h", "params_setup.h")]
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
        lib.emu_voxels.argtypes = [vp, vp, C.c_longlong, C.c_float, vp]; lib.emu_voxels.restype = None
        lib.emu_dense.argtypes = [vp, vp, vp, vp, vp, vp]; lib.emu_dense.restype = None
        _lib = lib
    return _lib


class EmuVoxelsVolume(emu_py.EmuVolume):
    """EmuVolume over the library that also has emu_voxels / emu_dense"""

    def __init__(self, **kw):
        lib = load()
        saved = emu_py._lib
        emu_py._lib = lib                      # EmuVolume.__init__ binds the library it loads
        try:
            super().__init__(**kw)
        finally:
            emu_py._lib = saved

    def containing_voxels(self, pts, min_size: float = -1.0) -> np.ndarray:
        xyz = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(xyz), VOXEL_DTYPE)
        self.lib.emu_voxels(self.h, xyz.ctypes.data, len(xyz), float(min_size), out.ctypes.data)
        return out

    def dense(self, box):
        b = np.asarray(box, np.int32)
        shape = tuple(int(b[a + 3] - b[a]) for a in range(3))
        d = np.empty(shape, np.float32); w = np.empty(shape, np.float32)
        rgb = np.empty(shape + (3,), np.uint8); level = np.empty(shape, np.int8)
        self.lib.emu_dense(self.h, b.ctypes.data, d.ctypes.data, w.ctypes.data, rgb.ctypes.data, level.ctypes.data)
        return {"d": d, "w": w, "rgb": rgb, "level": level}
