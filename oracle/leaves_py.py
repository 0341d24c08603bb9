"""ctypes binding of the oracle libraries with the leaf accessors (oracle/tsdf_oracle_leaves.h, built by oracle/leaves.mk):
"port" = the restatement (oracle/libtsdf_oracle_leaves.so), "reference" = the reference's own getVoxelCenters /
getOccupiedVoxelIndices (oracle/_ref/libcpu_tsdf_ref_leaves.so).  Each library carries the whole oracle C API as well.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle_py

HERE = os.path.dirname(os.path.abspath(__file__))
MK = os.path.join(HERE, "leaves.mk")
PORT_LIB = os.path.join(HERE, "libtsdf_oracle_leaves.so")
REF_LIB = os.path.join(HERE, "_ref", "libcpu_tsdf_ref_leaves.so")

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
    lib.orc_voxel_centers.argtypes = [vp, C.c_int, C.POINTER(vp)]; lib.orc_voxel_centers.restype = C.c_int64
    lib.orc_occupied_voxel_indices.argtypes = [vp, C.POINTER(vp)]; lib.orc_occupied_voxel_indices.restype = C.c_int64
    _libs[kind] = lib
    return lib


class LeavesOracleVolume(oracle_py.OracleVolume):
    """OracleVolume over a library that also has getVoxelCenters / getOccupiedVoxelIndices"""

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

    def _records(self, n, buf, dtype):
        out = np.empty((n, 3), dtype)
        if n:
            C.memmove(out.ctypes.data, buf.value, n * 12)
        return out

    def voxel_centers(self, nlevels: int = 4) -> np.ndarray:
        buf = C.c_void_p()
        n = self.lib.orc_voxel_centers(self.h, int(nlevels), C.byref(buf))
        return self._records(n, buf, np.float32)

    def occupied_voxel_indices(self) -> np.ndarray:
        buf = C.c_void_p()
        n = self.lib.orc_occupied_voxel_indices(self.h, C.byref(buf))
        return self._records(n, buf, np.int32)
