"""ctypes binding of the oracle libraries with the point lookup (oracle/tsdf_oracle_voxels.h, built by oracle/voxels.mk):
"port" = the restatement (oracle/libtsdf_oracle_voxels.so), "reference" = the reference's own
octree_->getContainingVoxel and node accessors (oracle/_ref/libcpu_tsdf_ref_voxels.so).  Each library carries the whole
oracle C API as well.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle_py

HERE = os.path.dirname(os.path.abspath(__file__))
MK = os.path.join(HERE, "voxels.mk")
PORT_LIB = os.path.join(HERE, "libtsdf_oracle_voxels.so")
REF_LIB = os.path.join(HERE, "_ref", "libcpu_tsdf_ref_voxels.so")

# orc_voxel = b200tsdf_voxel
VOXEL_DTYPE = np.dtype([("level", "<i4"), ("x", "<i4"), ("y", "<i4"), ("z", "<i4"),
                        ("cx", "<f4"), ("cy", "<f4"), ("cz", "<f4"), ("size", "<f4"),
                        ("d", "<f4"), ("w", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1"), ("has_children", "u1")])

_libs: dict[str, C.CDLL] = {}


def build(ref: bool = False) -> str:
    subprocess.run(["make", "-s", "-f", MK] + (["ref"] if ref else []), check=True)
    return REF_LIB if ref else PORT_LIB


def load(kind: str = "port") -> C.CDLL:
    if kind in _libs:
        return _libs[kind]
    if kind == "port":
        build()
    path = PORT_LIB if kind == "port" else REF_LIB
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    lib = C.CDLL(path)
    base = oracle_py.load("port")                    # the oracle C API: the same declarations
    for name in ("orc_default_config", "orc_create", "orc_destroy", "orc_reset", "orc_integrate", "orc_get_stats", "orc_query",
                 "orc_interpolate", "orc_render", "orc_mesh", "orc_save", "orc_dump_nodes", "orc_levels", "orc_voxel_center",
                 "orc_voxel_index", "orc_frustum_cull", "orc_dump_color_payload"):
        f, g = getattr(lib, name), getattr(base, name)
        f.argtypes, f.restype = g.argtypes, g.restype
    vp = C.c_void_p
    lib.orc_containing_voxels.argtypes = [vp, vp, C.c_int64, C.c_float, vp]
    lib.orc_containing_voxels.restype = None
    _libs[kind] = lib
    return lib


class VoxelsOracleVolume(oracle_py.OracleVolume):
    """OracleVolume over a library that also has the point lookup"""

    def __init__(self, kind: str = "port", **kw):
        lib = load(kind)
        saved = oracle_py._libs.get(kind)
        oracle_py._libs[kind] = lib                  # OracleVolume.__init__ binds the library oracle_py.load returns
        try:
            super().__init__(kind=kind, **kw)
        finally:
            if saved is None:
                del oracle_py._libs[kind]
            else:
                oracle_py._libs[kind] = saved

    def containing_voxels(self, pts, min_size: float = -1.0) -> np.ndarray:
        xyz = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(xyz), VOXEL_DTYPE)
        self.lib.orc_containing_voxels(self.h, xyz.ctypes.data, len(xyz), float(min_size), out.ctypes.data)
        return out
