"""Volumes, point sets and outputs for the point queries getFxn / getGradient / getHessian (query_point) and getTSDFValue
(interpolate_trilinearly): tests/test_queries.py, tests/test_queries_gpu.py, tools/make_query_pins.py.

The point sets sit where those routines branch: exactly on voxel centres and voxel faces, one ulp either side of them, in
the first and last three voxel layers of the grid, between leaves of different depths, and on NaN, infinities and
coordinates beyond 2^31 voxels.  Everything is float32 in the reference's order, generated from seeds and from the node dump
of the fused volume (finest-level leaves = the observed band).  Every backend (the restatement, the reference build, the host
emulation, the CUDA engine) is driven through `outputs(vol, points)`, where `vol` has query (pts, what, mode) ->
(val, grad, hess, ok) and interpolate (pts, valid_in) -> (val, valid).

tools/make_query_pins.py took 41 s on one core for all eight volumes on the reference build."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from cpu_tsdf_b200 import synth
from tests import dynamic_cases, general_cases
from tests.common import CAM, CFG_256, CFG_2048, frames
from tests.voxels import voxel_centers_1d

f32 = np.float32
WHATS = (1, 2, 4, 3, 7)
MODES = (0, 1)
VALID_INS = ("all", "none", "mix")


# ---- volumes ----------------------------------------------------------------------------------------------------------------
@dataclass
class Volume:
    id: str
    config: dict                                   # shared field names of OrcConfig, EmuVolume's and the engine's config
    frames: object                                 # () -> iterator of (pose, cloud)
    pool_log2: int = 17                            # hash pool of the emulation and the engine

    @property
    def res(self):
        return self.config["xres"]

    @property
    def size(self):
        return self.config["xsize"]


def _shape(res, size, cell):
    return dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy,
                max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)


def _shape_frames(size):
    scene = synth.Scene(room_half=min(1.3, size * 0.45), cam_radius=0.8)
    return lambda: frames(scene, 2, stride=6, noise_seed=9)


def _volumes():
    g1, g4, k1 = general_cases.CASES["G1"], general_cases.CASES["G4"], dynamic_cases.CASES["K1"]
    vs = [
        Volume("Q256", dict(CFG_256, integrate_color=1), lambda: frames(synth.S1, 5, stride=7, color=True, noise_seed=5)),
        Volume("Q256b", _shape(256, 2.7, 0.3), _shape_frames(2.7)),              # size / res is not exact in float
        Volume("Q512", _shape(512, 12.0, 0.5), _shape_frames(12.0)),             # coarse levels above the bricks
        Volume("Q1024", _shape(1024, 3.0, 0.5), _shape_frames(3.0), 19),         # 2.9 mm voxels
        Volume("Q2048", dict(CFG_2048, integrate_color=1),                       # the coarse cells are the root arrays
               lambda: frames(synth.S2, 2, stride=3, color=True, noise_seed=7, dropout=0.01), 18),
        Volume("Q4096", g4.config(), g4.frames, 19),                             # three tiers
        Volume("QK", k1.config(), k1.frames),                                    # pruned and re-split neighbourhoods
        Volume("QE", g1.config(), g1.frames),                                    # max_dist_pos != max_dist_neg
    ]
    return {v.id: v for v in vs}


VOLUMES = _volumes()
IDS = list(VOLUMES)


def fuse(vol, volume: Volume):
    for pose, cloud in volume.frames():
        vol.integrate(cloud, pose)
    return vol


# ---- the grid in float64, as getVoxelIndex / getVoxelCenter state it (tsdf_volume_octree.cpp:553-574) ----------------------------
def face_exact(size, res, idx):
    """float64 position of the face between voxels idx - 1 and idx"""
    s = np.float64(f32(size))
    return np.asarray(idx, np.float64) * s / np.float64(res) - s / 2.0


def face_floats(size, res, idx):
    """the float nearest to each face and, where the face is not a float, the neighbour on its other side (else the same float)"""
    e = face_exact(size, res, idx)
    near = e.astype(np.float32)
    d = e - near.astype(np.float64)
    other = np.where(d > 0, np.nextafter(near, f32(np.inf)), np.where(d < 0, np.nextafter(near, f32(-np.inf)), near))
    return near, other.astype(np.float32)


def index_expr(size, res, x):
    """getVoxelIndex's argument of floor (), in float64 as the reference evaluates it"""
    s = np.float64(f32(size))
    return (np.asarray(x, np.float64) + s / 2.0) / s * np.float64(res)


def tie_counts(size, res, pts):
    """Coordinates of `pts` on an exact tie, recomputed in float64: `centre` = equal to getVoxelCenter of the voxel they index
    (pt - centre == 0: the `<` of the half-voxel shift and sgn (0)), `face` = getVoxelIndex's floor () argument is an integer,
    `nonfinite` = NaN or infinite."""
    p = np.asarray(pts, np.float32)
    fin = np.isfinite(p)
    with np.errstate(invalid="ignore", over="ignore"):
        t = index_expr(size, res, np.where(fin, p, 0))
        inside = fin & (t >= 0) & (t < res)
        i = np.where(inside, np.floor(t), 0)
        centre = inside & (voxel_centers_1d(size, res, i) == p)
        face = fin & (t >= 0) & (t <= res) & (t == np.round(t))
    return {"centre": int(centre.sum()), "face": int(face.sum()), "nonfinite": int((~fin).sum())}


def border_layer_counts(size, res, pts):
    """points whose getVoxelIndex lies in voxel layers 0 (getTSDFValue refuses, getFxn may not), 1 and 2, res - 3 and res - 2,
    and res - 1, on any axis, and points outside the grid"""
    p = np.asarray(pts, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        i = np.floor(index_expr(size, res, p))
    inside = np.isfinite(p).all(1) & (i >= 0).all(1) & (i < res).all(1)
    lay = lambda *ls: int((inside & np.isin(i, ls).any(1)).sum())
    return {"layer0": lay(0), "layer1_2": lay(1, 2), "layer_m3_m2": lay(res - 3, res - 2), "layer_m1": lay(res - 1),
            "outside": int((~inside).sum())}


# ---- the node dump as a lookup: the leaf that holds each finest voxel ----------------------------------------------------------
class LeafIndex:
    """dump_nodes() of a fused volume (levels C .. L, every node) indexed by level and position"""

    def __init__(self, nodes, res):
        self.res, self.L = res, res.bit_length() - 1
        keys = nodes["keys"].astype(np.int64)
        self.C = int(keys[:, 0].min())
        self.level = {}
        for lv in range(self.C, self.L + 1):
            m = keys[:, 0] == lv
            code = (keys[m, 1] << (2 * lv)) | (keys[m, 2] << lv) | keys[m, 3]
            o = np.argsort(code)
            self.level[lv] = (code[o], nodes["dw"][m][o])

    def leaf(self, ijk):
        """(depth, d, w) of the leaf that holds each finest voxel of `ijk` [n, 3] (all inside the grid)"""
        ijk = np.asarray(ijk, np.int64)
        depth = np.full(len(ijk), -1, np.int64)
        dw = np.zeros((len(ijk), 2), np.float32)
        for lv in range(self.C, self.L + 1):
            q = ijk >> (self.L - lv)
            code = (q[:, 0] << (2 * lv)) | (q[:, 1] << lv) | q[:, 2]
            codes, vals = self.level[lv]
            if len(codes) == 0:
                break
            at = np.minimum(np.searchsorted(codes, code), len(codes) - 1)
            hit = codes[at] == code
            depth[hit] = lv
            dw[hit] = vals[at[hit]]
        assert (depth >= self.C).all()
        return depth, dw[:, 0], dw[:, 1]

    def finest_leaves(self):
        """positions [n, 3] of the finest-level nodes that were observed (w > 0): the band around the fused surface"""
        codes, vals = self.level[self.L]
        c = codes[vals[:, 1] > 0]
        m = (1 << self.L) - 1
        return np.stack([c >> (2 * self.L), (c >> self.L) & m, c & m], 1)

    def next_to_coarser(self):
        """(positions [n, 3], directions [n, 3]) of finest-level nodes whose face neighbour in that direction lies inside the grid
        and is held by a coarser leaf"""
        codes = self.level[self.L][0]
        m = (1 << self.L) - 1
        pos = np.stack([codes >> (2 * self.L), (codes >> self.L) & m, codes & m], 1)
        out_p, out_d = [], []
        for a in range(3):
            for s in (-1, 1):
                d = np.zeros(3, np.int64); d[a] = s
                nb = pos + d
                ok = (nb[:, a] >= 0) & (nb[:, a] < self.res)
                ncode = (nb[:, 0] << (2 * self.L)) | (nb[:, 1] << self.L) | nb[:, 2]
                ok &= codes[np.minimum(np.searchsorted(codes, ncode), len(codes) - 1)] != ncode
                out_p.append(pos[ok]); out_d.append(np.broadcast_to(d, (int(ok.sum()), 3)))
        return np.concatenate(out_p), np.concatenate(out_d)


def base_voxel(size, res, pts):
    """float64: the lower corner voxel of each point's 2x2x2 neighbourhood, clipped into the grid (the cell is ambiguous at a
    tie; the interpolant is continuous there)"""
    return np.clip(np.floor(index_expr(size, res, pts) - 0.5), 0, res - 2).astype(np.int64)


def neighbourhood_depths(index: LeafIndex, size, pts):
    """leaf depth of the eight voxels around each point: [n, 8]"""
    b = base_voxel(size, index.res, pts)
    return np.stack([index.leaf(b + np.array(o))[0] for o in np.ndindex(2, 2, 2)], 1)


def mixed_depth_count(index: LeafIndex, size, pts):
    d = neighbourhood_depths(index, size, pts)
    return int((d.min(1) != d.max(1)).sum())


# ---- float64 statement of what the queries compute, sharing no code with any backend -------------------------------------------
def trilinear64(index: LeafIndex, size, pts, with_gradient=False):
    """The trilinear interpolant of the leaf values at the eight finest-voxel centres around each point, in float64: what
    getTSDFValue returns, and getFxn in its finest-centre form (the two formulas are algebraically equal inside one cell).
    With with_gradient, also a central finite difference of the same cell's interpolant over a quarter voxel."""
    res = index.res
    p = np.asarray(pts, np.float64)
    b = base_voxel(size, res, p)
    c0 = np.stack([voxel_centers_1d(size, res, b[:, a]) for a in range(3)], 1).astype(np.float64)
    c1 = np.stack([voxel_centers_1d(size, res, b[:, a] + 1) for a in range(3)], 1).astype(np.float64)
    d = {o: index.leaf(b + np.array(o))[1].astype(np.float64) for o in np.ndindex(2, 2, 2)}

    def at(q):
        t = (q - c0) / (c1 - c0)
        s = np.zeros(len(q))
        for o, dv in d.items():
            w = np.ones(len(q))
            for a in range(3):
                w = w * (t[:, a] if o[a] else 1.0 - t[:, a])
            s += w * dv
        return s

    if not with_gradient:
        return at(p)
    h = (c1 - c0) / 4.0
    g = np.stack([(at(p + np.eye(3)[a] * h) - at(p - np.eye(3)[a] * h)) / (2.0 * h[:, a]) for a in range(3)], 1)
    return at(p), g


# ---- point sets ---------------------------------------------------------------------------------------------------------------
def _pick(rng, a, n):
    return a[rng.choice(len(a), min(n, len(a)), replace=False)]


def _near(rng, size, res, ijk):
    """random points within a voxel and a half of the centres of `ijk`"""
    c = np.stack([voxel_centers_1d(size, res, ijk[:, a]) for a in range(3)], 1).astype(np.float64)
    return (c + rng.uniform(-1.5, 1.5, c.shape) * (size / res)).astype(np.float32)


def _axes_masks(n):
    """for n points, which coordinates are pinned: a third each with one, two and three axes, rotating through the axes"""
    k = np.arange(n)
    count = k % 3 + 1
    first = (k // 3) % 3
    return np.stack([((np.arange(3)[None, :] - first[:, None]) % 3)[:, a] < count for a in range(3)], 1)


def point_sets(volume: Volume, nodes, seed=0) -> dict:
    """named [n, 3] float32 point sets for a fused volume whose dump_nodes() is `nodes`"""
    size, res = volume.size, volume.res
    rng = np.random.default_rng([seed, res, int(round(size * 1000))])
    index = LeafIndex(nodes, res)
    half = f32(size) / f32(2)
    vs = size / res
    band = index.finest_leaves()
    assert len(band) > 1000
    band = band[(band >= 3).all(1) & (band < res - 3).all(1)]
    sets = {}

    # random: near the fused surface plus uniform over a little more than the grid
    sets["random"] = np.concatenate([_near(rng, size, res, _pick(rng, band, 1500)),
                                     rng.uniform(-half * 1.05, half * 1.05, (1500, 3)).astype(np.float32)])

    # voxels around the fused surface and in empty space, for the centre and face sets
    vox = np.concatenate([_pick(rng, band, 900), rng.integers(3, res - 3, (300, 3))])
    pin = _axes_masks(len(vox))
    ctr = np.stack([voxel_centers_1d(size, res, vox[:, a]) for a in range(3)], 1)
    sets["centres"] = np.where(pin, ctr, _near(rng, size, res, vox)).astype(np.float32)
    near, other = (np.stack(x, 1) for x in zip(*(face_floats(size, res, vox[:, a]) for a in range(3))))
    loose = _near(rng, size, res, vox)
    sets["faces"] = np.concatenate([np.where(pin, near, loose), np.where(pin, other, loose)]).astype(np.float32)
    both = np.concatenate([sets["centres"], sets["faces"]])
    sets["ulp"] = np.concatenate([np.nextafter(both, f32(np.inf)), np.nextafter(both, f32(-np.inf))]).astype(np.float32)

    # border: on every face of the volume, voxel layers 0, 1, 2 and res-3, res-2, res-1 at their centres, quarter points and
    # faces, each also one ulp up and down; the other coordinates anywhere, or in a border layer too; then the corners
    vals = []
    for lay in (0, 1, 2, res - 3, res - 2, res - 1):
        c = voxel_centers_1d(size, res, [lay])[0]
        vals += [c, f32(c - 0.25 * vs), f32(c + 0.25 * vs), *face_floats(size, res, [lay])[0], *face_floats(size, res, [lay])[1]]
    vals += [half, -half]
    vals = np.array(vals, np.float32)
    vals = np.unique(np.concatenate([vals, np.nextafter(vals, f32(np.inf)), np.nextafter(vals, f32(-np.inf))]))
    border = []
    for a in range(3):
        for v in vals:
            q = rng.uniform(-half, half, (4, 3)).astype(np.float32)
            q[:, a] = v
            q[2:, (a + 1) % 3] = rng.choice(vals, 2)
            q[3, (a + 2) % 3] = rng.choice(vals)
            border.append(q)
    inner = np.nextafter(half, f32(0))
    corners = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float32)
    sets["border"] = np.concatenate(border + [corners * half, corners * inner]).astype(np.float32)

    # mixed: between a finest voxel and a face neighbour held by a coarser leaf
    pos, dirn = index.next_to_coarser()
    sel = rng.choice(len(pos), min(1500, len(pos)), replace=False)
    pos, dirn = pos[sel], dirn[sel]
    c = np.stack([voxel_centers_1d(size, res, pos[:, a]) for a in range(3)], 1).astype(np.float64)
    off = np.where(dirn != 0, dirn * rng.uniform(0.05, 0.95, (len(pos), 1)), rng.uniform(-0.45, 0.45, pos.shape))
    sets["mixed"] = (c + off * vs).astype(np.float32)

    # special: NaN, infinities, beyond 2^31 voxels, signed zeros, denormals, the floats just inside the faces
    nan, inf, den = f32(np.nan), f32(np.inf), f32(1e-45)
    x, y, z = (float(v) for v in sets["random"][0])
    sp = [[nan, y, z], [x, nan, z], [x, y, nan], [nan, nan, nan], [inf, y, z], [x, -inf, z], [x, y, inf], [-inf, -inf, -inf],
          [3e38, y, z], [x, -3e38, z], [x, y, 3e38], [-3e38, 3e38, -3e38], [1e10, y, z], [x, -1e10, z], [x, y, 1e10],
          [-1e10, -1e10, -1e10], [0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [0.0, -0.0, 0.0], [den, -den, den], [-den, den, 1e-39],
          [inner, y, z], [x, -inner, z], [x, y, inner], [-inner, -inner, -inner], [nan, inf, -0.0]]
    sets["special"] = np.array(sp, np.float32)
    return sets


# ---- outputs ------------------------------------------------------------------------------------------------------------------
def valid_in(kind, n):
    if kind == "mix":
        return (np.random.default_rng(n).random(n) < 0.7).astype(np.uint8)
    return np.full(n, 1 if kind == "all" else 0, np.uint8)


def query_bytes(what, val, grad, hess, ok):
    """the `ok` vector and the bits of every requested output at the ok points"""
    out = np.asarray(ok, bool).tobytes()
    for bit, a in ((1, val), (2, grad), (4, hess)):
        if what & bit:
            out += np.ascontiguousarray(a[ok]).view(np.uint32).tobytes()
    return out


def interp_bytes(val, valid):
    """the valid flags, the NaN mask and the bits of the values that are not NaN"""
    nan = np.isnan(val)
    return np.asarray(valid, bool).tobytes() + nan.tobytes() + np.ascontiguousarray(val[~nan]).view(np.uint32).tobytes()


def outputs(vol, volume: Volume, sets, index: LeafIndex = None) -> dict:
    """{name: bytes | number} for tests.common.digests: per set the points, the tie and border-layer counters recomputed in
    float64, and every call's outputs with its count of ok / valid / NaN results"""
    out = {}
    for name, pts in sets.items():
        out[f"{name}.pts"] = pts.tobytes()
        out[f"{name}.n"] = len(pts)
        for k, v in {**tie_counts(volume.size, volume.res, pts), **border_layer_counts(volume.size, volume.res, pts)}.items():
            out[f"{name}.{k}"] = v
        if name == "mixed" and index is not None:
            out["mixed.neighbourhoods_of_two_depths"] = mixed_depth_count(index, volume.size, pts)
        for mode in MODES:
            for what in WHATS:
                val, grad, hess, ok = vol.query(pts, what, mode)
                out[f"{name}.query_w{what}_m{mode}"] = query_bytes(what, val, grad, hess, ok)
                out[f"{name}.query_m{mode}.n_ok"] = int(ok.sum())
        for kind in VALID_INS:
            val, valid = vol.interpolate(pts, valid_in(kind, len(pts)))
            out[f"{name}.tsdf_{kind}"] = interp_bytes(val, valid)
            out[f"{name}.tsdf_{kind}.n_valid"], out[f"{name}.tsdf_{kind}.n_nan"] = int(valid.sum()), int(np.isnan(val).sum())
    return out


class OracleAdapter:
    """the restatement (kind "port") or the reference build (kind "reference") after the volume's frames"""

    def __init__(self, volume: Volume, kind="port"):
        from oracle.oracle_py import OracleVolume
        self.v = OracleVolume(kind=kind, **volume.config)
        self.v.reset()
        fuse(self.v, volume)

    def dump_nodes(self):
        return self.v.dump_nodes()

    def query(self, pts, what, mode):
        return self.v.query(pts, what, mode)

    def interpolate(self, pts, valid):
        return self.v.interpolate(pts, valid)


class EmuAdapter(OracleAdapter):
    """the host emulation of the engine's device code (tests/emu)"""

    def __init__(self, volume: Volume):
        from tests.emu.emu_py import EmuVolume
        self.v = EmuVolume(**volume.config, pool_log2=volume.pool_log2)
        self.v.reset()
        fuse(self.v, volume)
