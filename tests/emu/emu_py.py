"""ctypes wrapper of the host emulation of the engine's device code (tests/emu/emu.cpp).
TEST HARNESS ONLY — see the header of emu.cpp."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import Config

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu.so")
SRC = os.path.join(HERE, "emu.cpp")
CORE = os.path.join(HERE, "..", "..", "cpu_tsdf_b200", "csrc")


def build():
    deps = [SRC] + [os.path.join(CORE, f) for f in ("tsdf_core.cuh", "organize.cuh", "meshpost_core.cuh", "host_math.h", "params_setup.h")]
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
        lib.emu_dump_nodes.argtypes = [vp] + [vp] * 6; lib.emu_dump_nodes.restype = C.c_longlong
        lib.emu_query.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
        lib.emu_interpolate.argtypes = [vp, vp, C.c_int, vp, vp]
        lib.emu_render.argtypes = [vp, vp, C.c_int, vp, C.c_size_t, C.c_int, C.c_int, vp]
        lib.emu_mesh.argtypes = [vp, C.c_float, C.c_int, C.POINTER(vp), C.POINTER(vp)]; lib.emu_mesh.restype = C.c_longlong
        lib.emu_levels.argtypes = [vp, vp]
        lib.emu_frustum_cull.argtypes = [vp, vp, vp]
        lib.emu_organize.argtypes = [vp, C.c_size_t, C.c_size_t, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp, C.c_size_t, C.c_int]
        lib.emu_organize.restype = C.c_longlong
        lib.emu_mesh_flatten.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, vp, vp, vp, vp, vp]
        lib.emu_mesh_cleanup.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, C.c_int, vp, vp, vp, vp]
        _lib = lib
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class EmuVolume:
    def __init__(self, **kw):
        self.lib = load()
        import cpu_tsdf_b200 as pkg
        cfg = Config()
        # same defaults as b200tsdf_default_config
        cfg.xres = cfg.yres = cfg.zres = 512
        cfg.xsize = cfg.ysize = cfg.zsize = 3.0
        cfg.max_dist_pos = cfg.max_dist_neg = 0.03
        cfg.max_weight = 100
        cfg.min_sensor_dist, cfg.max_sensor_dist = 0.3, 3.0
        cfg.fx = cfg.fy = 525.0; cfg.cx, cfg.cy = 320, 240
        cfg.image_width, cfg.image_height = 640, 480
        cfg.max_cell_x = cfg.max_cell_y = cfg.max_cell_z = 0.5
        cfg.pool_log2 = 16
        cfg.shard_count = 1
        for i in range(4):
            cfg.global_transform[i * 5] = 1.0
        gt = kw.pop("global_transform", None)
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise AttributeError(k)
            setattr(cfg, k, v)
        if gt is not None:
            cfg.global_transform = (C.c_double * 16)(*np.asarray(gt, dtype=np.float64).reshape(16))
        self.cfg = cfg
        self.h = self.lib.emu_create(C.byref(cfg))

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.emu_destroy(self.h); self.h = None
        except Exception:
            pass

    def reset(self):
        rc = self.lib.emu_reset(self.h)
        assert rc == 0, rc

    def integrate(self, cloud, pose):
        cloud = np.ascontiguousarray(cloud, dtype=np.float32)
        H, W, nf = cloud.shape
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        rc = self.lib.emu_integrate(self.h, _ptr(cloud), nf * 4, 0, 16 if nf >= 5 else -1, W, H, _ptr(pose))
        assert rc == 0, rc

    def stats(self):
        o = np.zeros(3, np.int64)
        self.lib.emu_stats(self.h, _ptr(o))
        return {"n_updates": int(o[0]), "n_visits": int(o[1]), "n_culled": int(o[2])}

    def levels(self):
        o = np.zeros(4, np.int32)
        self.lib.emu_levels(self.h, _ptr(o))
        return tuple(int(v) for v in o)

    def dump_nodes(self):
        n = self.lib.emu_dump_nodes(self.h, None, None, None, None, None, None)
        assert n >= 0
        keys = np.empty((n, 4), np.int32); dw = np.empty((n, 2), np.float32); flags = np.empty(n, np.uint8)
        rgb = np.empty((n, 3), np.uint8); M = np.empty(n, np.float32); ns = np.empty(n, np.int32)
        self.lib.emu_dump_nodes(self.h, _ptr(keys), _ptr(dw), _ptr(flags), _ptr(rgb), _ptr(M), _ptr(ns))
        return {"keys": keys, "dw": dw, "split": flags, "rgb": rgb, "M": M, "ns": ns}

    def query(self, xyz, what=7, mode=0):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        n = len(xyz)
        val = np.full(n, np.nan, np.float32); grad = np.full((n, 3), np.nan, np.float32)
        hess = np.full((n, 3, 3), np.nan, np.float32); ok = np.zeros(n, np.uint8)
        self.lib.emu_query(self.h, _ptr(xyz), n, what, mode, _ptr(val), _ptr(grad), _ptr(hess), _ptr(ok))
        return val, grad, hess, ok.astype(bool)

    def interpolate(self, xyz, valid_in=True):
        """k_interpolate's routine; `valid_in` is one flag or one per point.  Returns (values, valid)."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        n = len(xyz)
        val = np.zeros(n, np.float32); ok = np.broadcast_to(np.asarray(valid_in, bool), (n,)).astype(np.uint8)
        self.lib.emu_interpolate(self.h, _ptr(xyz), n, _ptr(val), _ptr(ok))
        return val, ok.astype(bool)

    def render(self, pose, downsample=1, colored=False):
        W, H = self.cfg.image_width // downsample, self.cfg.image_height // downsample
        out = np.zeros((H, W, 12), np.float32)
        rgb = np.zeros((H, W, 3), np.uint8) if colored else None
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        self.lib.emu_render(self.h, _ptr(pose), downsample, _ptr(out), 48, 0, 16, _ptr(rgb))
        return (out, rgb) if colored else out

    def mesh(self, w_min=2.5, color_mode=0):
        pv, pc = C.c_void_p(), C.c_void_p()
        n = self.lib.emu_mesh(self.h, w_min, color_mode, C.byref(pv), C.byref(pc))
        verts = np.empty((n, 3), np.float32); rgb = None
        if n:
            C.memmove(verts.ctypes.data, pv.value, n * 12)
            if pc.value:
                rgb = np.empty((n, 3), np.uint8); C.memmove(rgb.ctypes.data, pc.value, n * 3)
        return verts, rgb

    def frustum_cull(self, pose):
        c = self.levels()[0]
        n = 1 << c
        mask = np.zeros((n, n, n), np.uint8)
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        kept = self.lib.emu_frustum_cull(self.h, _ptr(pose), _ptr(mask))
        return mask, kept


def organize(points, intr, width, height, *, rgba_off=-1, cloud_units=1.0, zero_nans=False, world_to_camera=None,
             out_stride=32, out_rgba_off=16):
    lib = load()
    pts = np.ascontiguousarray(points, dtype=np.float32)
    intr = np.asarray(intr, np.float32)
    out = np.full((height, width, out_stride // 4), 7.0, np.float32)       # pre-filled: padding must come back zero
    tf = None if world_to_camera is None else np.ascontiguousarray(world_to_camera, dtype=np.float64)
    filled = lib.emu_organize(_ptr(pts), pts.shape[0], pts.shape[1] * 4, 0, rgba_off, _ptr(intr), width, height,
                              float(cloud_units), int(zero_nans), _ptr(tf), _ptr(out), out_stride, out_rgba_off)
    return out, int(filled)


def _mesh_call(fn, verts, tris, *args, extra=()):
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3); tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    ov = np.zeros_like(verts); ot = np.zeros_like(tris)
    nv = C.c_size_t(0); nt = C.c_size_t(0)
    fn(_ptr(verts), len(verts), _ptr(tris), len(tris), *args, _ptr(ov), C.byref(nv), _ptr(ot), C.byref(nt), *extra)
    return ov[:nv.value].copy(), ot[:nt.value].copy()


def flatten_vertices(verts, tris, min_dist=0.0001, return_rounds=False):
    rounds = C.c_int(0)
    out = _mesh_call(load().emu_mesh_flatten, verts, tris, C.c_float(min_dist), extra=(C.byref(rounds),))
    return out + (rounds.value,) if return_rounds else out


def cleanup_mesh(verts, tris, face_dist=0.02, min_neighbors=5):
    return _mesh_call(load().emu_mesh_cleanup, verts, tris, C.c_float(face_dist), int(min_neighbors))
