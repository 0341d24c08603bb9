"""ctypes binding of the CPU oracle (oracle/libtsdf_oracle.so, or oracle/_ref/libcpu_tsdf_ref.so).

TEST INFRASTRUCTURE ONLY.  Import this from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs — never from the cpu_tsdf_b200 package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PORT_LIB = os.path.join(HERE, "libtsdf_oracle.so")
REF_LIB = os.path.join(HERE, "_ref", "libcpu_tsdf_ref.so")


class OrcConfig(C.Structure):
    _fields_ = [
        ("xres", C.c_int32), ("yres", C.c_int32), ("zres", C.c_int32),
        ("xsize", C.c_float), ("ysize", C.c_float), ("zsize", C.c_float),
        ("max_dist_pos", C.c_float), ("max_dist_neg", C.c_float), ("max_weight", C.c_float),
        ("min_sensor_dist", C.c_float), ("max_sensor_dist", C.c_float),
        ("max_cell_x", C.c_float), ("max_cell_y", C.c_float), ("max_cell_z", C.c_float),
        ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
        ("image_width", C.c_int32), ("image_height", C.c_int32),
        ("integrate_color", C.c_int32), ("num_threads", C.c_int32),
        ("global_transform", C.c_double * 16),
        ("color_mode", C.c_int32), ("reserved_", C.c_int32),
    ]


class OrcStats(C.Structure):
    _fields_ = [
        ("n_add_observation", C.c_int64), ("n_node_visits", C.c_int64), ("n_presplit", C.c_int64),
        ("n_culled_cells", C.c_int64), ("n_nodes", C.c_int64),
        ("t_presplit", C.c_double), ("t_cull", C.c_double), ("t_update", C.c_double),
        ("n_prune_existing", C.c_int64), ("n_prune_resplit", C.c_int64),
    ]


def build(ref: bool = False) -> str:
    """(Re)build the oracle library with oracle/Makefile; returns the path."""
    target = ["ref"] if ref else []
    subprocess.run(["make", "-s", "-C", HERE] + target, check=True)
    return REF_LIB if ref else PORT_LIB


_libs: dict[str, C.CDLL] = {}


REFPROG_LIB = os.path.join(HERE, "_ref", "libcpu_tsdf_refprog.so")


def load_prog(kind: str = "port") -> C.CDLL:
    """The program-side functions (organise / flattenVertices / cleanupMesh): "port" = oracle/prog_oracle.cpp inside the restatement
    library, "reference" = the reference's own text of src/prog/integrate.cpp (oracle/_ref/libcpu_tsdf_refprog.so, `make refprog`)."""
    if kind == "port":
        return load("port")
    if "refprog" in _libs:
        return _libs["refprog"]
    if not os.path.exists(REFPROG_LIB):
        raise FileNotFoundError(REFPROG_LIB)
    lib = C.CDLL(REFPROG_LIB)
    vp = C.c_void_p
    lib.orc_organize.argtypes = [vp, C.c_size_t, C.c_size_t, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp]
    lib.orc_organize.restype = C.c_int64
    lib.orc_flatten_vertices.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, vp, vp, vp, vp]
    lib.orc_cleanup_mesh.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, C.c_int, vp, vp, vp, vp]
    _libs["refprog"] = lib
    return lib


def load(kind: str = "port") -> C.CDLL:
    """kind = "port" (the restatement) or "reference" (the reference's own sources, oracle/_ref)."""
    if kind in _libs:
        return _libs[kind]
    path = PORT_LIB if kind == "port" else REF_LIB
    if kind == "port":
        build()                      # make: a no-op when the library is newer than its sources
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    lib = C.CDLL(path)
    vp = C.c_void_p
    lib.orc_default_config.argtypes = [C.POINTER(OrcConfig)]
    lib.orc_create.argtypes = [C.POINTER(OrcConfig)]; lib.orc_create.restype = vp
    lib.orc_destroy.argtypes = [vp]
    lib.orc_reset.argtypes = [vp]
    lib.orc_integrate.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    lib.orc_get_stats.argtypes = [vp, C.POINTER(OrcStats)]
    lib.orc_query.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    lib.orc_interpolate.argtypes = [vp, vp, C.c_int, vp, vp]
    lib.orc_render.argtypes = [vp, vp, C.c_int, vp, C.c_size_t, C.c_int, C.c_int, vp]
    lib.orc_mesh.argtypes = [vp, C.c_float, C.c_int, C.POINTER(vp), C.POINTER(vp)]; lib.orc_mesh.restype = C.c_int64
    lib.orc_save.argtypes = [vp, C.c_char_p]
    lib.orc_dump_nodes.argtypes = [vp, vp, vp, vp, vp, vp, vp]; lib.orc_dump_nodes.restype = C.c_int64
    lib.orc_levels.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.orc_voxel_center.argtypes = [vp, C.c_int64, C.c_int64, C.c_int64, vp]
    lib.orc_voxel_index.argtypes = [vp, C.c_float, C.c_float, C.c_float, vp]
    lib.orc_frustum_cull.argtypes = [vp, vp, vp]
    lib.orc_dump_color_payload.argtypes = [vp, vp]; lib.orc_dump_color_payload.restype = C.c_int64
    if kind == "port":               # the program-side restatement (oracle/prog_oracle.cpp) exists in the port only
        lib.orc_organize.argtypes = [vp, C.c_size_t, C.c_size_t, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp]
        lib.orc_organize.restype = C.c_int64
        lib.orc_flatten_vertices.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, vp, vp, vp, vp]
        lib.orc_cleanup_mesh.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.c_float, C.c_int, vp, vp, vp, vp]
    _libs[kind] = lib
    return lib


def organize(points: np.ndarray, intr, width: int, height: int, *, rgba_off: int = -1, cloud_units: float = 1.0,
             zero_nans: bool = False, world_to_camera=None, kind: str = "port"):
    """integrate.cpp:548-607 — z-buffer an unorganised cloud ([n, k] float32 rows, xyz first, colour bytes at
    rgba_off) into [height, width, 8] float32 rows in pcl::PointXYZRGBA layout.  Returns (organized, n_filled)."""
    lib = load_prog(kind)
    pts = np.ascontiguousarray(points, dtype=np.float32)
    intr = np.asarray(intr, np.float32)
    out = np.zeros((height, width, 8), np.float32)
    tf = None if world_to_camera is None else np.ascontiguousarray(world_to_camera, dtype=np.float64)
    filled = lib.orc_organize(_ptr(pts), pts.shape[0], pts.shape[1] * 4, 0, rgba_off, _ptr(intr), width, height,
                              float(cloud_units), int(zero_nans), _ptr(tf), _ptr(out))
    return out, int(filled)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class OracleVolume:
    """Mirror of cpu_tsdf::TSDFVolumeOctree over the oracle C API."""

    def __init__(self, kind: str = "port", **kw):
        self.lib = load(kind)
        self.cfg = OrcConfig()
        self.lib.orc_default_config(C.byref(self.cfg))
        gt = kw.pop("global_transform", None)
        for k, v in kw.items():
            if not hasattr(self.cfg, k):
                raise AttributeError(k)
            setattr(self.cfg, k, v)
        if gt is not None:
            self.cfg.global_transform = (C.c_double * 16)(*np.asarray(gt, dtype=np.float64).reshape(16))
        self.h = self.lib.orc_create(C.byref(self.cfg))
        self._keep = None

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.orc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def reset(self):
        return self.lib.orc_reset(self.h)

    def integrate(self, cloud: np.ndarray, pose: np.ndarray):
        cloud = np.ascontiguousarray(cloud, dtype=np.float32)
        H, W, nf = cloud.shape
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        rc = self.lib.orc_integrate(self.h, _ptr(cloud), nf * 4, 0, 16 if nf >= 8 else -1, W, H, _ptr(pose))
        assert rc == 0
        return rc

    def stats(self) -> OrcStats:
        s = OrcStats()
        self.lib.orc_get_stats(self.h, C.byref(s))
        return s

    def levels(self):
        a, b = C.c_int(), C.c_int()
        self.lib.orc_levels(self.h, C.byref(a), C.byref(b))
        return a.value, b.value

    def query(self, xyz: np.ndarray, what: int = 7, mode: int = 0):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        n = len(xyz)
        val = np.full(n, np.nan, np.float32); grad = np.full((n, 3), np.nan, np.float32)
        hess = np.full((n, 3, 3), np.nan, np.float32); ok = np.zeros(n, np.uint8)
        self.lib.orc_query(self.h, _ptr(xyz), n, what, mode, _ptr(val), _ptr(grad), _ptr(hess), _ptr(ok))
        return val, grad, hess, ok.astype(bool)

    def interpolate(self, xyz: np.ndarray, valid_in=True):
        """getTSDFValue = interpolateTrilinearly (cpp:454-541).  Returns (values, valid) with valid starting as `valid_in`
        (one flag, or one per point)."""
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        n = len(xyz)
        val = np.zeros(n, np.float32); ok = np.broadcast_to(np.asarray(valid_in, bool), (n,)).astype(np.uint8)
        self.lib.orc_interpolate(self.h, _ptr(xyz), n, _ptr(val), _ptr(ok))
        return val, ok.astype(bool)

    def render(self, pose: np.ndarray, downsample: int = 1, colored: bool = False):
        W, H = self.cfg.image_width // downsample, self.cfg.image_height // downsample
        out = np.zeros((H, W, 12), np.float32)
        rgb = np.zeros((H, W, 3), np.uint8) if colored else None
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        self.lib.orc_render(self.h, _ptr(pose), downsample, _ptr(out), 48, 0, 16, _ptr(rgb))
        return (out, rgb) if colored else out

    def mesh(self, w_min: float = 2.5, color_mode: int = 0):
        pv, pc = C.c_void_p(), C.c_void_p()
        n = self.lib.orc_mesh(self.h, w_min, color_mode, C.byref(pv), C.byref(pc))
        verts = np.empty((n, 3), np.float32)
        rgb = None
        if n:
            C.memmove(verts.ctypes.data, pv.value, n * 12)
            if pc.value:
                rgb = np.empty((n, 3), np.uint8)
                C.memmove(rgb.ctypes.data, pc.value, n * 3)
        return verts, rgb

    def save(self, path: str):
        return self.lib.orc_save(self.h, path.encode())

    def dump_nodes(self):
        n = self.lib.orc_dump_nodes(self.h, None, None, None, None, None, None)
        keys = np.empty((n, 4), np.int32); dw = np.empty((n, 2), np.float32); flags = np.empty(n, np.uint8)
        rgb = np.empty((n, 3), np.uint8); M = np.empty(n, np.float32); ns = np.empty(n, np.int32)
        self.lib.orc_dump_nodes(self.h, _ptr(keys), _ptr(dw), _ptr(flags), _ptr(rgb), _ptr(M), _ptr(ns))
        out = {"keys": keys, "dw": dw, "split": flags, "rgb": rgb, "M": M, "ns": ns}
        if self.cfg.integrate_color and self.cfg.color_mode == 1:
            payload = np.zeros((n, 4), np.float32)                 # RGBNormalized: r_n_, g_n_, b_n_, i_
            assert self.lib.orc_dump_color_payload(self.h, _ptr(payload)) == n
            out["rgbn"] = payload
        return out

    def voxel_center(self, x, y, z):
        o = np.empty(3, np.float32)
        self.lib.orc_voxel_center(self.h, x, y, z, _ptr(o))
        return o

    def voxel_index(self, x, y, z):
        o = np.empty(3, np.int32)
        ok = self.lib.orc_voxel_index(self.h, x, y, z, _ptr(o))
        return o, bool(ok)

    def frustum_cull(self, pose):
        c, _ = self.levels()
        n = 1 << c
        mask = np.zeros((n, n, n), np.uint8)
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        kept = self.lib.orc_frustum_cull(self.h, _ptr(pose), _ptr(mask))
        return mask, kept


def _mesh_call(fn, verts, tris, *args):
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3); tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    ov = np.zeros_like(verts); ot = np.zeros_like(tris)
    nv = C.c_size_t(0); nt = C.c_size_t(0)
    fn(_ptr(verts), len(verts), _ptr(tris), len(tris), *args, _ptr(ov), C.byref(nv), _ptr(ot), C.byref(nt))
    return ov[:nv.value].copy(), ot[:nt.value].copy()


def flatten_vertices(verts, tris, min_dist=0.0001, kind: str = "port"):
    """flattenVertices, integrate.cpp:103-150 -> (vertices [n,3], triangles [m,3])"""
    return _mesh_call(load_prog(kind).orc_flatten_vertices, verts, tris, C.c_float(min_dist))


def cleanup_mesh(verts, tris, face_dist=0.02, min_neighbors=5, kind: str = "port"):
    """cleanupMesh, integrate.cpp:152-214"""
    return _mesh_call(load_prog(kind).orc_cleanup_mesh, verts, tris, C.c_float(face_dist), int(min_neighbors))
