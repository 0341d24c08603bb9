"""Point sets, dense boxes and digests for getContainingVoxel and the dense crop (tests/test_voxels.py, tests/test_voxels_gpu.py,
tools/make_voxel_pins.py).  Everything is float32 arithmetic in the reference's order, generated from seeds."""
from __future__ import annotations

import hashlib

import numpy as np

f32 = np.float32


def node_center(size: float, level: int, x: int) -> np.float32:
    """OctreeNode::getCenter on one axis: ctr -/+ size/4 from the root, size halving (octree.cpp:244-266)"""
    c, off = f32(0.0), f32(size) * f32(0.25)
    for i in range(level - 1, -1, -1):
        c = c + off if (x >> i) & 1 else c - off
        off = off * f32(0.5)
    return f32(c)


def level_size(size: float, level: int) -> np.float32:
    s = f32(size)
    for _ in range(level):
        s = s * f32(0.5)
    return f32(s)


def voxel_centers_1d(size: float, res: int, idx) -> np.ndarray:
    """getVoxelCenter on one axis (tsdf_volume_octree.cpp:553-560): float ((i + 0.5) * size / res - float (size / 2.0))"""
    s = np.float64(f32(size))
    voff = np.float64(f32(s / 2.0))
    i = np.asarray(idx, np.float64)
    return ((i + 0.5) * s / np.float64(res) - voff).astype(np.float32)


def float_descent_bits(size: float, levels: int, v: np.ndarray) -> np.ndarray:
    """the child bit chosen at each level by the float descent, (v - ctr) > 0 in float32, for every value of v: [levels, len(v)]"""
    v = np.asarray(v, np.float32)
    c = np.zeros_like(v)
    off = f32(size) * f32(0.25)
    out = np.zeros((levels, len(v)), np.uint8)
    for lv in range(levels):
        bit = (v - c) > 0
        out[lv] = bit
        c = np.where(bit, c + off, c - off).astype(np.float32)
        off = off * f32(0.5)
    return out


def point_sets(size: float, finest: int, seed: int = 0) -> dict:
    """named [n, 3] float32 point sets: uniform, on splitting planes, on and one ulp outside the faces, NaN and -0.0"""
    rng = np.random.default_rng(seed)
    half = f32(size) / f32(2)
    sets = {"uniform": rng.uniform(-half * 1.02, half * 1.02, (4000, 3)).astype(np.float32)}
    planes = []
    for lv in range(finest):
        n = 1 << lv
        xs = sorted(set(int(v) for v in rng.integers(0, n, 6))) if n > 6 else range(n)
        for x in xs:
            c = node_center(size, lv, x)
            q = rng.uniform(-half, half, (4, 3)).astype(np.float32)
            q[0, 0] = c; q[1, 1] = c; q[2, 2] = c; q[3, :] = c
            planes.append(q)
    sets["planes"] = np.concatenate(planes).astype(np.float32)
    out = np.nextafter(half, f32(np.inf), dtype=np.float32)
    faces = []
    for a in range(3):
        for v in (half, -half, out, -out):
            q = rng.uniform(-half, half, (3, 3)).astype(np.float32)
            q[:, a] = v
            faces.append(q)
    faces.append(np.array([[half, half, half], [-half, -half, -half], [out, 0, 0], [0, 0, -out]], np.float32))
    sets["faces"] = np.concatenate(faces).astype(np.float32)
    nan = np.float32(np.nan)
    sets["special"] = np.array([[0, 0, nan], [nan, 0, 0], [0, nan, 0.1], [nan, nan, 0.2], [-0.0, -0.0, -0.0], [-0.0, 0.0, -0.0],
                                [0.0, -0.0, 0.3], [nan, 0.4, -0.4]], np.float32)
    return sets


def min_sizes(size: float, finest: int) -> list:
    """-1, 0, each level's exact node size, values between sizes and one above the root size"""
    out = [-1.0, 0.0]
    for lv in range(finest + 1):
        s = level_size(size, lv)
        out.append(float(s))
        out.append(float(s * f32(0.75)))
    out.append(float(f32(size) * f32(1.5)))
    return out


def dense_from_lookups(lookup, size: float, res: int, box) -> dict:
    """the dense crop restated: the lookup (min_size -1) at getVoxelCenter (i, j, k) of every voxel of the box"""
    i0, j0, k0, i1, j1, k1 = (int(v) for v in box)
    ci, cj, ck = (voxel_centers_1d(size, res, np.arange(a, b)) for a, b in ((i0, i1), (j0, j1), (k0, k1)))
    pts = np.stack(np.meshgrid(ci, cj, ck, indexing="ij"), axis=-1).reshape(-1, 3)
    rec = lookup(pts)
    shape = (i1 - i0, j1 - j0, k1 - k0)
    assert (rec["level"] >= 0).all()
    return {"d": rec["d"].reshape(shape), "w": rec["w"].reshape(shape),
            "rgb": np.stack([rec["r"], rec["g"], rec["b"]], -1).reshape(shape + (3,)), "level": rec["level"].astype(np.int8).reshape(shape)}


def digest(a: np.ndarray) -> list:
    a = np.ascontiguousarray(a)
    return [int(a.shape[0]) if a.ndim else 1, hashlib.sha256(a.tobytes()).hexdigest()]


def lookup_outputs(lookup, size: float, finest: int, seed: int = 0, sizes=None) -> dict:
    """every point set at every min_size: name -> structured array"""
    out = {}
    sets = point_sets(size, finest, seed)
    for ms in (min_sizes(size, finest) if sizes is None else sizes):
        for name, pts in sets.items():
            out[f"{name}@{ms!r}"] = lookup(pts, ms)
    return out
