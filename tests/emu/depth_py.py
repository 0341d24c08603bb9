"""ctypes wrapper of the host emulation of k_depth_unproject (tests/emu/depth_emu.cpp).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import DEPTH_F32, DEPTH_U16

HERE = os.path.dirname(os.path.abspath(__file__))
CORE = os.path.join(HERE, "..", "..", "cpu_tsdf_b200", "csrc")
LIB = os.path.join(HERE, "libemu_depth.so")
SRC = os.path.join(HERE, "depth_emu.cpp")


def build():
    deps = [SRC] + [os.path.join(CORE, f) for f in ("tsdf_core.cuh", "organize.cuh", "depth.cuh")]
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
        lib.emu_depth_to_cloud.argtypes = [vp, C.c_int, C.c_float, vp, C.c_int, C.c_int, vp, vp]
        _lib = lib
    return _lib


def depth_to_pixels(depth: np.ndarray, intrinsics, rgb=None, depth_scale=1e-3) -> np.ndarray:
    """[H, W, 4] uint32: the 16-byte pixels {x, y, z, bgra} that k_depth_unproject writes, computed on the host"""
    d = np.ascontiguousarray(depth)
    fmt = DEPTH_U16 if d.dtype == np.uint16 else DEPTH_F32
    assert d.dtype in (np.uint16, np.float32) and d.ndim == 2
    H, W = d.shape
    intr = np.array([np.float32(v) for v in intrinsics], np.float32)
    c = None if rgb is None else np.ascontiguousarray(rgb, dtype=np.uint8)
    out = np.empty((H, W, 4), np.uint32)
    load().emu_depth_to_cloud(d.ctypes.data, fmt, float(np.float32(depth_scale)), None if c is None else c.ctypes.data, W, H,
                              intr.ctypes.data, out.ctypes.data)
    return out


def cloud_pixels(cloud: np.ndarray) -> np.ndarray:
    """the 16-byte pixels of a depth_to_cloud result ([H, W, 8] float32): its words 0-2 and 4, as uint32"""
    w = np.ascontiguousarray(cloud).view(np.uint32)
    return np.ascontiguousarray(w[..., [0, 1, 2, 4]])
