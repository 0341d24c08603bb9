"""Scenes that change while they are fused, for the parity tests of pruning and re-splitting.

Every other stream in the suite fuses a static scene, so the surface is refined and almost never carved away.  Here a
sphere and an axis-aligned box move, shrink, vanish and come back inside the room, so that nodes whose children existed
before a frame have all their children pruned (impl/tsdf_volume_octree.hpp:136-141), and often split again in the same
updateVoxel call (hpp:161-188).  The flat layout never releases a brick, so a later re-split lands on storage that was
carved before: it must be exactly fresh (DESIGN.md §2).

The frames follow synth.make_frame's conventions (organized W x H cloud in the sensor frame, NaN = invalid, PCL b,g,r,a
colour bytes, the same noise model and colour pattern); synth.py itself stays as bench.py uses it.  Every backend is
driven through `outputs(case, vol)` with the adapters of tests/general_cases.py."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from cpu_tsdf_b200 import synth
from tests.common import nan_fixed
from tests import general_cases
from tests.general_cases import OracleAdapter, random_poses  # noqa: F401  (OracleAdapter serves these cases as it is)


@dataclass
class Objects:
    """what stands in the room during one frame: a sphere (centre, radius) and an axis-aligned box (centre, half sides)"""
    sphere: tuple | None = None
    box: tuple | None = None


def ray_depth(room_half, objects: Objects, pose, cam: synth.Camera):
    """float64 z-depth of every pixel (inf where nothing is hit) and the ray directions, as synth._ray_depth computes them"""
    u = np.arange(cam.width, dtype=np.float64)
    v = np.arange(cam.height, dtype=np.float64)
    xn, yn = np.broadcast_arrays((u[None, :] - cam.cx) / cam.fx, (v[:, None] - cam.cy) / cam.fy)
    d_w = np.stack([xn, yn, np.ones_like(xn)], axis=-1) @ pose[:3, :3].T        # z component 1 in the camera: t is z-depth
    o = pose[:3, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        t_axis = (np.where(d_w > 0, room_half, -room_half) - o) / d_w
    t = np.where(np.isfinite(t_axis) & (t_axis > 0), t_axis, np.inf).min(axis=-1)
    if objects.sphere is not None:
        c, r = np.asarray(objects.sphere[0], np.float64), float(objects.sphere[1])
        oc = o - c
        a = (d_w * d_w).sum(-1)
        b = 2.0 * (d_w @ oc)
        disc = b * b - 4 * a * (float(oc @ oc) - r * r)
        with np.errstate(invalid="ignore"):
            ts = (-b - np.sqrt(np.where(disc > 0, disc, np.nan))) / (2 * a)
        t = np.where((disc > 0) & (ts > 0) & (ts < t), ts, t)
    if objects.box is not None:
        lo = np.asarray(objects.box[0], np.float64) - np.asarray(objects.box[1], np.float64)
        hi = np.asarray(objects.box[0], np.float64) + np.asarray(objects.box[1], np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            t1, t2 = (lo - o) / d_w, (hi - o) / d_w
        tn = np.where(np.isnan(t1), -np.inf, np.minimum(t1, t2)).max(axis=-1)
        tf = np.where(np.isnan(t1), np.inf, np.maximum(t1, t2)).min(axis=-1)
        t = np.where((tn <= tf) & (tn > 0) & (tn < t), tn, t)
    return t, xn, yn, d_w, o


def make_frame(room_half, objects: Objects, pose, cam: synth.Camera, *, color=False, noise_seed=None, frame=0):
    """synth.make_frame for a scene with moving objects: [H, W, 4] float32 (xyz, 1) or, with colour, [H, W, 8] (xyz, 1,
    then the bytes b,g,r,a in float slot 4); depth noise sigma(z) = 0.0012 + 0.0019 (z - 0.4)^2 m when noise_seed is given"""
    t, xn, yn, d_w, o = ray_depth(room_half, objects, pose, cam)
    if noise_seed is not None:
        rng = np.random.default_rng([noise_seed, frame])
        t = t + rng.standard_normal(t.shape) * (0.0012 + 0.0019 * (t - 0.4) ** 2)
    valid = np.isfinite(t) & (t > 0)
    out = np.empty((cam.height, cam.width, 8 if color else 4), np.float32)
    t32 = np.where(valid, t, np.nan)
    out[..., 0] = (xn * t32).astype(np.float32)
    out[..., 1] = (yn * t32).astype(np.float32)
    out[..., 2] = t32.astype(np.float32)
    out[..., 3] = 1.0
    if color:
        cell = np.floor((o + d_w * np.where(valid, t, 0.0)[..., None]) / 0.032).astype(np.int64)
        par = (cell.sum(-1) & 1).astype(np.uint8)
        rgba = np.zeros((cam.height, cam.width, 4), np.uint8)
        rgba[..., 2] = np.where(par == 1, 220, 40) + (np.mod(cell[..., 0], 8) * 4).astype(np.uint8)
        rgba[..., 1] = np.where(par == 1, 180, 60) + (np.mod(cell[..., 1], 8) * 4).astype(np.uint8)
        rgba[..., 0] = np.where(par == 1, 90, 200) + (np.mod(cell[..., 2], 8) * 4).astype(np.uint8)
        rgba[..., 3] = 255
        out[..., 4] = rgba.view(np.float32)[..., 0]
        out[..., 5:] = 0.0
    return np.ascontiguousarray(out)


@dataclass
class Case:
    id: str
    res: int
    size: float
    room_half: float
    poses: list                                    # one camera->world pose per frame
    objects: list                                  # one Objects per frame
    cam: synth.Camera = field(default_factory=synth.Camera)
    color: bool = False
    color_mode: int = 0                            # 1: RGBNormalized
    track_variance: bool = False                   # the engine's M / nsample storage (the restatement always keeps it)
    noise_seed: int | None = 11
    params: dict = field(default_factory=dict)     # max_weight, truncation, sensor bounds
    per_frame: bool = False                        # digests of the nodes after every frame
    render_ds: tuple = (2,)
    mesh_wmin: tuple = (0.0,)

    def config(self):
        """the configuration shared by OracleVolume, EmuVolume and the engine's b200tsdf_config (same field names)"""
        c = self.cam
        return dict(xres=self.res, yres=self.res, zres=self.res, xsize=self.size, ysize=self.size, zsize=self.size,
                    fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, image_width=c.width, image_height=c.height,
                    integrate_color=int(self.color), color_mode=self.color_mode, **self.params)

    def frames(self):
        for f, (pose, obj) in enumerate(zip(self.poses, self.objects)):
            yield pose, make_frame(self.room_half, obj, pose, self.cam, color=self.color, noise_seed=self.noise_seed, frame=f)


S1_POSE = synth.orbit_pose(synth.S1, 0, 100)       # at (1, 0, 0) looking at the room's centre
ORIGIN = (0.0, 0.0, 0.0)


def shrinking(r0, step, n):
    return [Objects(sphere=(ORIGIN, r0 - step * f)) for f in range(n)]


def wall_box(pose, room_half, half, slide, n):
    """a box against the wall that pose's optical axis meets, sliding `slide` metres per frame along that wall towards the
    room's centre line"""
    o, d = pose[:3, 3], pose[:3, 2]
    with np.errstate(divide="ignore"):
        ta = (np.where(d > 0, room_half, -room_half) - o) / d
    k = int(np.argmin(np.where(ta > 0, ta, np.inf)))
    hit = o + d * ta[k]
    half = np.asarray(half, np.float64)
    centre = hit.copy()
    centre[k] = np.sign(d[k]) * (room_half - half[k])
    along = (k + 1) % 3
    step = -slide if hit[along] > 0 else slide
    return [Objects(box=(tuple(centre + np.eye(3)[along] * (step * f)), tuple(half))) for f in range(n)]


def _cases():
    cs = []
    mw1 = dict(max_weight=1.0)
    # K1: 256^3 / 3 m, a shrinking sphere seen from a fixed camera.  Weight cap 1: every free-space observation moves d halfway
    # to +1, so a node reads empty (d >= 0.99) after about seven of them
    cs.append(Case("K1", 256, 3.0, 1.4, [S1_POSE] * 10, shrinking(0.45, 0.04, 10), color=True, params=mw1))
    # K2: 512^3 / 3 m, a sphere for three frames and then none; the variance state must return to zero on prune
    gone = [Objects(sphere=(ORIGIN, 0.35))] * 3 + [Objects()] * 9
    cs.append(Case("K2", 512, 3.0, 1.4, [S1_POSE] * 12, gone, track_variance=True, params=mw1))
    # K3: 256^3, a shrinking sphere with the RGBNormalized payload
    cs.append(Case("K3", 256, 3.0, 1.4, [S1_POSE] * 8, shrinking(0.45, 0.04, 8), color=True, color_mode=1, params=mw1))
    # K4: 2048^3 / 10 m interior, colour, a box sliding along the wall in view of a look-at camera with pitch and roll
    p4 = random_poses(synth.S2, 10, 401)
    cs.append(Case("K4", 2048, 10.0, 2.0, p4, wall_box(p4[0], 2.0, (0.3, 0.3, 0.3), 0.12, 10), color=True,
                   params=dict(max_weight=2.0), render_ds=(4,)))
    # K5: 4096^3 / 10 m, coarse levels above the supercells: a box for two frames, then gone (with a weight cap of 1 a node
    # needs about seven free-space observations before it reads empty)
    p5 = random_poses(synth.S2, 10, 402)
    box = wall_box(p5[0], 2.0, (0.3, 0.3, 0.3), 0.0, 2)
    cs.append(Case("K5", 4096, 10.0, 2.0, p5, box + [Objects()] * 8, params=mw1, render_ds=(4,), mesh_wmin=()))
    # K6: carve, then bring the object back: the re-split lands on bricks whose hash slots stayed claimed
    back = [Objects(sphere=(ORIGIN, 0.45))] * 3 + [Objects()] * 3 + [Objects(sphere=(ORIGIN, 0.45))] * 3
    cs.append(Case("K6", 256, 3.0, 1.4, [S1_POSE] * 9, back, color=True, params=mw1, per_frame=True))
    return {c.id: c for c in cs}


CASES = _cases()
IDS = list(CASES)


class EmuAdapter(general_cases.EmuAdapter):
    """the host emulation (tests/emu), with the case's variance storage"""

    def __init__(self, case: Case, pool_log2=17):
        from tests.emu.emu_py import EmuVolume
        self.v = EmuVolume(**case.config(), track_variance=int(case.track_variance), pool_log2=pool_log2)
        self.v.reset()


def node_digest_bytes(d):
    return d["keys"].tobytes() + d["split"].tobytes() + d["dw"].view(np.uint32).tobytes()


def outputs(case: Case, vol):
    """Everything the parity tests compare, as {name: array | number}: levels, nodes, colour, variance state, the RGBNormalized
    payload, addObservation counts per frame (backends that count them), per-frame nodes (K6), a render and a mesh."""
    upd, per = [], []
    for pose, cloud in case.frames():
        vol.integrate(cloud, pose)
        upd.append(vol.n_updates())
        if case.per_frame:
            per.append(node_digest_bytes(vol.dump_nodes()))
    d = vol.dump_nodes()
    out = {"levels": np.array(vol.levels()[:2], np.int64), "keys": d["keys"], "split": d["split"],
           "dw": d["dw"].view(np.uint32)}
    if upd[0] is not None:
        out["n_updates"] = np.array(upd, np.int64)
    for i, b in enumerate(per):
        out[f"frame{i}_nodes"] = b
    if case.color:
        out["rgb"] = d["rgb"]
    if case.track_variance:
        out["M"], out["ns"] = d["M"].view(np.uint32), d["ns"]
    if case.color_mode == 1:
        out["rgbn"] = d["rgbn"].view(np.uint32)
    rpose = case.poses[-1]
    for ds in case.render_ds:
        r, c = vol.render(rpose, ds, case.color)
        out[f"render{ds}_xyz"], out[f"render{ds}_n"] = nan_fixed(r[..., :3]), nan_fixed(r[..., 4:7])
        if case.color:
            out[f"render{ds}_rgb"] = c
    for wmin in case.mesh_wmin:
        v, col = vol.mesh(wmin, 1 if case.color else 0)
        out[f"mesh{wmin:g}_n"], out[f"mesh{wmin:g}"] = len(v), np.asarray(v, np.float32).reshape(-1, 3).view(np.uint32)
        if case.color:
            out[f"mesh{wmin:g}_rgb"] = col
    return out


def event_counts(case: Case):
    """the restatement's prune events over the stream: (pre-existing children pruned, pruned and re-split in the same call)"""
    from oracle.oracle_py import OracleVolume
    v = OracleVolume(**case.config())
    v.reset()
    n = [0, 0]
    for pose, cloud in case.frames():
        v.integrate(cloud, pose)
        s = v.stats()
        n[0] += s.n_prune_existing
        n[1] += s.n_prune_resplit
    return tuple(n)
