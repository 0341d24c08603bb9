"""ctypes wrapper of the host emulation of the tracking kernels (tests/emu/track_emu.cpp, which compiles emu.cpp with them
added).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import TRACK_ITER_DTYPE, Config, TrackParams, TrackResult
from tests.emu import depth_py, emu_py

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu_track.so")
SRC = os.path.join(HERE, "track_emu.cpp")


def build():
    deps = [SRC, emu_py.SRC] + [os.path.join(emu_py.CORE, f) for f in ("tsdf_core.cuh", "organize.cuh", "meshpost_core.cuh", "host_math.h",
                                                                         "params_setup.h", "depth.cuh", "track.cuh")]
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
        lib.emu_stats.argtypes = [vp, vp]
        lib.emu_levels.argtypes = [vp, vp]
        lib.emu_dump_nodes.argtypes = [vp] + [vp] * 6; lib.emu_dump_nodes.restype = C.c_longlong
        lib.emu_query.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
        tp, tr = C.POINTER(TrackParams), C.POINTER(TrackResult)
        lib.track_run.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, tp, tr, vp]
        lib.track_samples_dump.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, tp, vp, vp, vp, vp, vp]
        lib.track_sums_once.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, tp, vp]
        lib.track_solve6.argtypes = [vp, C.c_double, vp, vp]
        lib.track_exp.argtypes = [vp, vp, vp]
        _lib = lib
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def as_cloud(frame, intrinsics=None, depth_scale=1e-3):
    """(pixels, stride, xyz_off) of a frame as the device reads it: an organised cloud [H, W, nf] float32 as it is, or a
    depth map ([H, W] uint16 / float32) as the 16-byte pixels k_depth_unproject writes"""
    f = np.asarray(frame)
    if f.ndim == 2:
        return np.ascontiguousarray(depth_py.depth_to_pixels(f, intrinsics, None, depth_scale)), 16, 0
    f = np.ascontiguousarray(f, dtype=np.float32)
    return f, f.shape[2] * 4, 0


class TrackEmuVolume(emu_py.EmuVolume):
    """EmuVolume with the tracking kernels' emulation"""

    def __init__(self, **kw):
        lib = load()
        saved = emu_py._lib
        emu_py._lib = lib                      # EmuVolume.__init__ binds the library it loads
        try:
            super().__init__(**kw)
        finally:
            emu_py._lib = saved

    def intrinsics(self):
        return (self.cfg.fx, self.cfg.fy, self.cfg.cx, self.cfg.cy)

    def track(self, frame, pose0, params=None, depth_scale=1e-3):
        """(pose, result) as TSDFVolumeOctree.trackDepth / trackCloudDevice return them"""
        prm = TrackParams.default() if params is None else params
        pts, stride, off = as_cloud(frame, self.intrinsics(), depth_scale)
        H, W = pts.shape[:2]
        pose = np.ascontiguousarray(pose0, dtype=np.float64)
        res = TrackResult()
        log = np.zeros(max(1, sum(prm.iters[:prm.levels])), TRACK_ITER_DTYPE)
        self.lib.track_run(self.h, _ptr(pts), stride, off, W, H, _ptr(pose), C.byref(prm), C.byref(res), _ptr(log))
        return np.array(res.pose_c2w, np.float64).reshape(4, 4), {
            "status": int(res.status), "iters": list(res.iters), "inliers": int(res.inliers), "rms": float(res.rms),
            "A": np.array(res.A, np.float64).reshape(6, 6), "b": np.array(res.b, np.float64), "log": log[:res.n_log].copy()}

    def samples(self, frame, pose, stride, params=None):
        """every sample at `pose`: dict of q [n, 3], r [n], g [n, 3], wlo [n], finite / ok / inlier [n] bool, and (u, v)"""
        prm = TrackParams.default() if params is None else params
        pts, st, off = as_cloud(frame, self.intrinsics())
        H, W = pts.shape[:2]
        cw, ch = -(-W // stride), -(-H // stride)
        n = cw * ch
        q = np.full((n, 3), np.nan, np.float32); r = np.full(n, np.nan, np.float32); g = np.full((n, 3), np.nan, np.float32)
        wlo = np.full(n, np.nan, np.float32); fl = np.zeros(n, np.uint8)
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        got = self.lib.track_samples_dump(self.h, _ptr(pts), st, off, W, H, _ptr(pose), stride, C.byref(prm), _ptr(q), _ptr(r), _ptr(g),
                                          _ptr(wlo), _ptr(fl))
        assert got == n
        j = np.arange(n)
        return {"q": q, "r": r, "g": g, "wlo": wlo, "finite": (fl & 1) > 0, "ok": (fl & 2) > 0, "inlier": (fl & 4) > 0,
                "u": (j % cw) * stride, "v": (j // cw) * stride}

    def sums(self, frame, pose, stride, params=None):
        prm = TrackParams.default() if params is None else params
        pts, st, off = as_cloud(frame, self.intrinsics())
        H, W = pts.shape[:2]
        out = np.zeros(30, np.float64)
        self.lib.track_sums_once(self.h, _ptr(pts), st, off, W, H, _ptr(np.ascontiguousarray(pose, dtype=np.float64)), stride,
                                 C.byref(prm), _ptr(out))
        return out


def solve6(A, lam, b):
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64); x = np.zeros(6)
    ok = load().track_solve6(_ptr(A), float(lam), _ptr(b), _ptr(x))
    return x, bool(ok)


def se3_exp_left(xi, T):
    xi = np.ascontiguousarray(xi, np.float64); T = np.ascontiguousarray(T, np.float64); out = np.zeros((4, 4))
    load().track_exp(_ptr(xi), _ptr(T), _ptr(out))
    return out
