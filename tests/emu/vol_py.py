"""ctypes wrapper of the host emulation of the .vol writer and parser (tests/emu/vol_emu.cpp, which compiles emu.cpp with
emu_vol_body and emu_vol_parse added).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import Config
from tests.emu import emu_py

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu_vol.so")
SRC = os.path.join(HERE, "vol_emu.cpp")


def build():
    deps = [SRC, emu_py.SRC] + [os.path.join(emu_py.CORE, f) for f in ("tsdf_core.cuh", "vol_io.cuh", "organize.cuh", "meshpost_core.cuh", "host_math.h", "params_setup.h")]
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
        lib.emu_vol_body.argtypes = [vp, vp]; lib.emu_vol_body.restype = C.c_longlong
        lib.emu_vol_parse.argtypes = [vp, vp, C.c_size_t, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
        _lib = lib
    return _lib


class EmuVolVolume(emu_py.EmuVolume):
    """EmuVolume over the library that also has the .vol writer and parser"""

    def __init__(self, **kw):
        lib = load()
        saved = emu_py._lib
        emu_py._lib = lib                      # EmuVolume.__init__ binds the library it loads
        try:
            super().__init__(**kw)
        finally:
            emu_py._lib = saved

    def body(self) -> bytes:
        n = self.lib.emu_vol_body(self.h, None)
        rb = 43 if self.cfg.integrate_color else 40
        out = np.empty(n * rb, np.uint8)
        self.lib.emu_vol_body(self.h, out.ctypes.data_as(C.c_void_p))
        return out.tobytes()

    def parse(self, body: bytes, rgb: bool):
        """(status, records of the tree or -1, out-of-domain count): status 1 placed, 0 refused (nothing placed)"""
        buf = np.frombuffer(body, np.uint8).copy() if body else np.zeros(1, np.uint8)
        n, ood = C.c_longlong(), C.c_longlong()
        st = self.lib.emu_vol_parse(self.h, buf.ctypes.data_as(C.c_void_p), len(body), int(rgb), C.byref(n), C.byref(ood))
        return st, n.value, ood.value
