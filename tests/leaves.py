"""getVoxelCenters / getOccupiedVoxelIndices restated over a node dump.  TEST INFRASTRUCTURE ONLY.

Octree::getLeaves (octree.cpp:99-109, :608-617) walks depth first, children in index order (x high bit, then y, z), and
emits a node of depth >= 1 when it has no children or its depth is `nlevels`, never going below that depth (nlevels < 0:
no limit; nlevels == 0: the root alone).  Every node above the coarse depth C exists and has children (Octree::init), so
for 0 <= nlevels < C the result is all 8^nlevels nodes of that depth.  Otherwise it is read off the dump of every node at
depth >= C that the restatement, the reference build (oracle/_ref), the host emulation and the engine all export
(level, x, y, z, {d, w}, has-children), in the reference's order: the selected nodes do not overlap, so the
bit-interleaved coordinates of their first finest voxel order them depth first.

getVoxelCenters returns OctreeNode::getCenter of each node: the centre accumulated at split time, ctr -/+ size/4 per
level from the root at (0,0,0) (octree.cpp:244-266), replayed here in float32.  getOccupiedVoxelIndices
(tsdf_volume_octree.cpp:590-609) keeps the leaves (nlevels = -1) with w > 0 && fabs (d) < 1 and maps each centre through
getVoxelIndex (cpp:562-574): floor (((double) x + size / 2.0) / size * res)."""
from __future__ import annotations

import hashlib

import numpy as np


def center1d(size: float, level: int, coords: np.ndarray) -> np.ndarray:
    c = np.zeros(len(coords), np.float32)
    off = np.float32(np.float32(size) * np.float32(0.25))
    coords = np.asarray(coords, np.int64)
    for i in range(level - 1, -1, -1):
        bit = ((coords >> i) & 1).astype(bool)
        c = np.where(bit, c + off, c - off).astype(np.float32)
        off = np.float32(off * np.float32(0.5))
    return c


def order_key(L: int, level: np.ndarray, x: np.ndarray, y: np.ndarray, z: np.ndarray) -> np.ndarray:
    sh = (L - np.asarray(level, np.int64))
    X, Y, Z = (np.asarray(a, np.int64) << sh for a in (x, y, z))
    k = np.zeros(len(sh), np.uint64)
    for l in range(L - 1, -1, -1):
        k = (k << np.uint64(3)) | (((X >> l) & 1) << 2).astype(np.uint64) | (((Y >> l) & 1) << 1).astype(np.uint64) | ((Z >> l) & 1).astype(np.uint64)
    return k


def _centres(size, level, x, y, z):
    level = np.asarray(level)
    out = np.empty((len(level), 3), np.float32)
    for lv in np.unique(level):
        m = level == lv
        for a, c in enumerate((x, y, z)):
            out[m, a] = center1d(size, int(lv), np.asarray(c)[m])
    return out


def voxel_index(size: float, res: int, xyz: np.ndarray) -> np.ndarray:
    ds = np.float64(np.float32(size))
    return np.floor((xyz.astype(np.float64) + ds / 2.0) / ds * np.float64(res)).astype(np.int32)


def leaves(dump: dict, coarse: int, finest: int, size: float, res: int, nlevels: int, occupied: bool = False) -> np.ndarray:
    """[N, 3] float32 centres (or int32 voxel indices when `occupied`) in the reference's order."""
    if not occupied and nlevels >= 0 and (nlevels < coarse or nlevels == 0):
        i = np.arange(8 ** nlevels, dtype=np.int64)
        x = np.zeros_like(i); y = np.zeros_like(i); z = np.zeros_like(i)
        for l in range(nlevels - 1, -1, -1):
            c = (i >> (3 * l)) & 7
            x = (x << 1) | (c >> 2); y = (y << 1) | ((c >> 1) & 1); z = (z << 1) | (c & 1)
        return _centres(size, np.full(len(i), nlevels), x, y, z)
    keys = np.asarray(dump["keys"]); level = keys[:, 0]
    split = np.asarray(dump["split"]).astype(bool)
    sel = level >= 1
    if nlevels >= 0:
        sel &= level <= nlevels
    sel &= ~split | (level == nlevels)
    if occupied:
        d, w = np.asarray(dump["dw"], np.float32).T
        sel &= (w > 0) & (np.abs(d) < 1)
    k = keys[sel]
    order = np.argsort(order_key(finest, k[:, 0], k[:, 1], k[:, 2], k[:, 3]), kind="stable")
    k = k[order]
    c = _centres(size, k[:, 0], k[:, 1], k[:, 2], k[:, 3])
    return voxel_index(size, res, c) if occupied else c


def nlevels_sweep(coarse: int, finest: int):
    return sorted({-1, 0, 1, coarse - 1, coarse, coarse + 1, finest - 1, finest, finest + 3})


def leaf_outputs(dump: dict, coarse: int, finest: int, size: float, res: int) -> dict:
    """every getVoxelCenters of the sweep and getOccupiedVoxelIndices, as arrays"""
    out = {}
    for n in nlevels_sweep(coarse, finest):
        out[f"centers{n}"] = leaves(dump, coarse, finest, size, res, n)
    out["occupied"] = leaves(dump, coarse, finest, size, res, -1, occupied=True)
    return out


def digest(outputs: dict) -> dict:
    """{name: [count, SHA-256 of the exact bytes]}: the form stored in tests/golden/leaf_pins.json"""
    return {k: [int(len(v)), hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest()] for k, v in outputs.items()}
