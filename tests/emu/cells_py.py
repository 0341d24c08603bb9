"""ctypes wrapper of the host emulation of the change epochs and of the cell-restricted mesh (tests/emu/cells_emu.cpp, which
compiles emu.cpp with them added).  TEST HARNESS ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import Config
from tests.emu import emu_py

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libemu_cells.so")
SRC = os.path.join(HERE, "cells_emu.cpp")


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
        lib.emu_levels.argtypes = [vp, vp]
        lib.emu_stats.argtypes = [vp, vp]
        lib.emu_dump_nodes.argtypes = [vp] + [vp] * 6; lib.emu_dump_nodes.restype = C.c_longlong
        lib.emu_frustum_cull.argtypes = [vp, vp, vp]
        lib.cells_create.restype = vp
        lib.cells_destroy.argtypes = [vp]
        lib.cells_reset.argtypes = [vp, vp]
        lib.cells_integrate.argtypes = [vp, vp, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        lib.cells_edits.argtypes = [vp, vp, vp, C.c_longlong, C.c_float, vp, vp, vp]; lib.cells_edits.restype = C.c_longlong
        lib.cells_changed.argtypes = [vp, vp, C.c_ulonglong, vp]; lib.cells_changed.restype = C.c_ulonglong
        lib.cells_mesh.argtypes = [vp, C.c_float, C.c_int, vp, C.POINTER(vp), C.POINTER(vp), vp]; lib.cells_mesh.restype = C.c_longlong
        _lib = lib
    return _lib


class CellsEmuVolume(emu_py.EmuVolume):
    """EmuVolume whose reset, frames and node writes keep the engine's change epochs"""

    def __init__(self, **kw):
        lib = load()
        saved = emu_py._lib
        emu_py._lib = lib                      # EmuVolume.__init__ binds the library it loads
        try:
            super().__init__(**kw)
        finally:
            emu_py._lib = saved
        self.epochs = lib.cells_create()

    def __del__(self):
        try:
            if getattr(self, "epochs", None):
                self.lib.cells_destroy(self.epochs); self.epochs = None
        except Exception:
            pass
        super().__del__()

    def reset(self):
        rc = self.lib.cells_reset(self.h, self.epochs)
        assert rc == 0, rc

    def integrate(self, cloud, pose):
        cloud = np.ascontiguousarray(cloud, dtype=np.float32)
        H, W, nf = cloud.shape
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        rc = self.lib.cells_integrate(self.h, self.epochs, cloud.ctypes.data, nf * 4, 0, 16 if nf >= 5 else -1, W, H, pose.ctypes.data)
        assert rc == 0, rc

    def set_containing_voxels(self, pts, d, w, min_size: float = -1.0) -> np.ndarray:
        xyz = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
        dd = np.ascontiguousarray(np.broadcast_to(np.asarray(d, np.float32), (len(xyz),)))
        ww = np.ascontiguousarray(np.broadcast_to(np.asarray(w, np.float32), (len(xyz),)))
        status = np.zeros(len(xyz), np.uint8)
        self.lib.cells_edits(self.h, self.epochs, xyz.ctypes.data, len(xyz), float(min_size), dd.ctypes.data, ww.ctypes.data,
                             status.ctypes.data)
        return status


def ncells(vol):
    return 1 << (3 * vol.levels()[0])


def changed_cells(vol, since):
    """(now, mask) as b200tsdf_changed_cells"""
    mask = np.zeros(ncells(vol), np.uint8)
    now = vol.lib.cells_changed(vol.h, vol.epochs, int(since), mask.ctypes.data)
    return int(now), mask


def mesh_cells(vol, w_min, color_mode, mask=None):
    """(verts [N,3] float32, rgb [N,3] uint8 or None, cell_nverts int64[8^C]) as b200tsdf_mesh_cells_device"""
    counts = np.zeros(ncells(vol), np.int64)
    m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    pv, pc = C.c_void_p(), C.c_void_p()
    n = vol.lib.cells_mesh(vol.h, w_min, color_mode, None if m is None else m.ctypes.data, C.byref(pv), C.byref(pc),
                           counts.ctypes.data)
    verts = np.empty((n, 3), np.float32); rgb = np.empty((n, 3), np.uint8) if color_mode else None
    if n:
        C.memmove(verts.ctypes.data, pv.value, n * 12)
        if color_mode:
            C.memmove(rgb.ctypes.data, pc.value, n * 3)
    return verts, rgb, counts


def morton_cells(ncells):
    """the cells in the mesh's order: perm[k] = the layout index ((x n + y) n + z) of the k-th cell in depth-first (Morton)
    order, x high"""
    C3 = int(ncells).bit_length() - 1
    k = np.arange(ncells, dtype=np.int64)
    x = np.zeros_like(k); y = np.zeros_like(k); z = np.zeros_like(k)
    for l in range(C3 // 3 - 1, -1, -1):
        c = (k >> (3 * l)) & 7
        x = (x << 1) | (c >> 2); y = (y << 1) | ((c >> 1) & 1); z = (z << 1) | (c & 1)
    n = 1 << (C3 // 3)
    return (x * n + y) * n + z


def splice(old, old_counts, new, new_counts, mask):
    """the mesh whose cell c is new's run of c where mask[c], else old's run of c, cells in Morton order
    (IncrementalMesh.update); counts and mask in the cell layout"""
    perm = morton_cells(len(mask))
    sel = np.asarray(mask, bool)[perm]
    oc, nc = np.asarray(old_counts)[perm], np.asarray(new_counts)[perm]
    counts = np.where(sel, nc, oc)
    excl = lambda c: np.concatenate(([0], np.cumsum(c)[:-1]))
    base = np.where(sel, len(old) + excl(nc), excl(oc))
    cell = np.repeat(np.arange(len(counts)), counts)
    idx = base[cell] + np.arange(counts.sum()) - excl(counts)[cell]
    out_counts = np.empty_like(counts); out_counts[perm] = counts
    return np.concatenate((old, new))[idx], out_counts


def runs(a, counts):
    """the per-cell runs of a mesh array, as a list indexed by cell (layout index)"""
    perm = morton_cells(len(counts))
    parts = np.split(a, np.cumsum(np.asarray(counts)[perm])[:-1])
    out = [None] * len(counts)
    for k, c in enumerate(perm):
        out[c] = parts[k]
    return out
