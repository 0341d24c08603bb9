"""General-input cases for the parity tests: look-at poses with pitch and roll, cameras other than the 525 / 319.5 / 239.5
one, asymmetric truncation, sensor clipping, a non-integer weight cap, a wide strip image, exact-tie geometry and a
truncation limit outside the range where the brick kernels' division is exact.

Every backend (the restatement, the reference build, the host emulation, the CUDA engine) is driven through the same
`outputs(case, vol)`, where `vol` is a small adapter over that backend (OracleAdapter, EmuAdapter here; the engine's adapter
lives in tests/test_general_geometry_gpu.py).  The outputs are compared through tests.common.digests."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from cpu_tsdf_b200 import synth
from tests.common import nan_fixed

TUM = synth.Camera(fx=517.3, fy=516.5, cx=318.6, cy=255.3, width=640, height=480)


def look_at_pose(eye, target, roll=0.0):
    """camera->world 4x4 (float64) in the synth convention (x right, y down = world +y when level, z forward) for a camera at
    `eye` looking at `target`, turned by `roll` radians about its viewing axis."""
    eye = np.asarray(eye, np.float64)
    fwd = np.asarray(target, np.float64) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross([0.0, 1.0, 0.0], fwd)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    c, s = math.cos(roll), math.sin(roll)
    pose = np.eye(4)
    pose[:3, 0] = c * right + s * down
    pose[:3, 1] = -s * right + c * down
    pose[:3, 2] = fwd
    pose[:3, 3] = eye
    return pose


def random_poses(scene: synth.Scene, n, seed):
    """n look-at poses with yaw, pitch and roll along a short random walk (consecutive views overlap, so weights above 1
    occur): the eye is inside the room and outside the sphere, the target is near the room's centre (S1: the sphere is in
    view) or beyond the eye (interior scenes: a wall is in view), roll up to +-40 degrees."""
    rng = np.random.default_rng(seed)
    R = scene.room_half
    while True:
        eye = rng.uniform(-0.6 * R, 0.6 * R, 3)
        if np.linalg.norm(eye) > scene.sphere_radius + 0.35:
            break
    target = rng.normal(scale=0.15 * R, size=3)
    out = []
    while len(out) < n:
        e = eye + rng.normal(scale=0.03 * R, size=3)
        t = target + rng.normal(scale=0.05 * R, size=3)
        if np.linalg.norm(e) < scene.sphere_radius + 0.3 or np.abs(e).max() > 0.7 * R:
            continue
        if scene.outward:
            t = e + (e - t)
        out.append(look_at_pose(e, t, rng.uniform(-0.7, 0.7)))
    return out


def axis_pose(perm, signs, t):
    """camera->world pose whose rotation is a signed permutation of the axes (column k = signs[k] * e_perm[k])"""
    pose = np.eye(4)
    pose[:3, :3] = 0.0
    for k in range(3):
        pose[perm[k], k] = signs[k]
    assert abs(np.linalg.det(pose[:3, :3]) - 1.0) < 1e-12
    pose[:3, 3] = t
    return pose


@dataclass
class Case:
    id: str
    res: int
    size: float
    cam: synth.Camera
    scene: synth.Scene
    poses: list
    color: bool = False
    noise_seed: int | None = None
    dropout: float = 0.0
    params: dict = field(default_factory=dict)     # max_dist_pos / _neg, max_weight, min_ / max_sensor_dist
    repeat: int = 1                                # each frame fused this many times in a row
    cull_poses: list = field(default_factory=list)
    render_ds: tuple = (1, 2, 3)
    mesh_wmin: tuple = (0.0, 2.0)

    def config(self):
        """the configuration shared by OracleVolume, EmuVolume and the engine's b200tsdf_config (same field names)"""
        c = self.cam
        return dict(xres=self.res, yres=self.res, zres=self.res, xsize=self.size, ysize=self.size, zsize=self.size,
                    fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, image_width=c.width, image_height=c.height,
                    integrate_color=int(self.color), **self.params)

    def frames(self):
        for f, pose in enumerate(self.poses):
            cloud = synth.make_frame(self.scene, pose, self.cam, color=self.color, noise_seed=self.noise_seed, frame=f,
                                     dropout=self.dropout)
            for _ in range(self.repeat):
                yield pose, cloud


S1, S2 = synth.S1, synth.S2
ROOM1 = synth.Scene(room_half=1.0, cam_radius=0.5, sphere=False)          # walls on node boundaries of a 4 m grid


def _cases():
    cs = []
    # (G1 and G3 have a multiple of four frames: tests/test_general_geometry_gpu.py fuses them in four graph-replayed batches)
    cs.append(Case("G1", 256, 3.0, TUM, S1, random_poses(S1, 8, 101), color=True, noise_seed=5, dropout=0.02,
                   params=dict(max_dist_pos=0.05, max_dist_neg=0.02), cull_poses=random_poses(S1, 3, 901)))
    cs.append(Case("G2", 512, 3.0, synth.Camera(525.0, 525.0, 320.0, 240.0), S1, random_poses(S1, 3, 102), noise_seed=6,
                   cull_poses=random_poses(S1, 3, 902)))
    cs.append(Case("G3", 2048, 10.0, TUM, S2, random_poses(S2, 4, 103), color=True, noise_seed=7,
                   cull_poses=random_poses(S2, 3, 903), render_ds=(2, 3, 4)))
    cs.append(Case("G4", 4096, 10.0, TUM, S2, random_poses(S2, 2, 104), noise_seed=8,
                   cull_poses=random_poses(S2, 3, 904), render_ds=(2, 3, 4)))
    clip = dict(min_sensor_dist=0.5, max_sensor_dist=1.2, max_weight=2.5)
    cs.append(Case("G5a", 256, 3.0, synth.Camera(262.5, 262.5, 159.5, 119.5, 320, 240), S1, random_poses(S1, 4, 105),
                   color=True, noise_seed=9, params=clip, cull_poses=random_poses(S1, 3, 905)))
    cs.append(Case("G5b", 256, 3.0, synth.Camera(525.0, 525.0, 321.0, 239.5, 643, 479), S1, random_poses(S1, 4, 106),
                   noise_seed=10, params=clip, cull_poses=random_poses(S1, 3, 906)))
    cs.append(Case("G6", 256, 3.0, synth.Camera(4096.0, 128.0, 4095.5, 31.5, 8192, 64), S1, random_poses(S1, 3, 107),
                   noise_seed=11, cull_poses=random_poses(S1, 3, 907), render_ds=(2, 3, 4)))
    # exact ties: axis-aligned poses with dyadic translations, walls on node planes, no noise
    tie_poses = [axis_pose((0, 1, 2), (1, 1, 1), (0.25, -0.125, -0.5)),
                 axis_pose((2, 1, 0), (1, 1, -1), (-0.375, 0.0625, 0.125)),
                 axis_pose((0, 2, 1), (-1, 1, 1), (0.125, -0.5, 0.25))]
    cs.append(Case("T1", 256, 4.0, synth.Camera(512.0, 512.0, 320.0, 240.0), ROOM1, tie_poses + tie_poses[:1],
                   params=dict(max_dist_pos=1 / 32, max_dist_neg=1 / 32), cull_poses=tie_poses))
    # outside the range where the brick kernels' division is exact: the weighted sum overflows to inf and is then divided
    cs.append(Case("D1", 512, 3.0, synth.Camera(525.0, 525.0, 320.0, 240.0), S1, random_poses(S1, 1, 108), repeat=10,
                   params=dict(max_dist_pos=10.0, max_dist_neg=1.2e-38), render_ds=(), mesh_wmin=()))
    return {c.id: c for c in cs}


CASES = _cases()
IDS = list(CASES)


def outputs(case: Case, vol):
    """Everything the parity tests compare, as {name: array | number}: levels, nodes, n_add_observation per frame, cull masks,
    renders (the colour variant when colour is fused) and meshes in the reference's order."""
    upd = []
    for pose, cloud in case.frames():
        vol.integrate(cloud, pose)
        upd.append(vol.n_updates())
    d = vol.dump_nodes()
    out = {"levels": np.array(vol.levels()[:2], np.int64), "keys": d["keys"], "split": d["split"],
           "dw": d["dw"].view(np.uint32)}
    if upd[0] is not None:                         # (the reference build does not count addObservation calls)
        out["n_updates"] = np.array(upd, np.int64)
    if case.color:
        out["rgb"] = d["rgb"]
    for i, pose in enumerate(case.cull_poses):
        out[f"cull{i}"] = vol.cull(pose).astype(np.uint8)
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


class OracleAdapter:
    """the restatement (kind "port") or the reference build (kind "reference")"""

    def __init__(self, case: Case, kind="port"):
        from oracle.oracle_py import OracleVolume
        self.v = OracleVolume(kind=kind, **case.config())
        self.v.reset()
        self.counts = kind == "port"

    def integrate(self, cloud, pose):
        self.v.integrate(cloud, pose)

    def n_updates(self):
        return self.v.stats().n_add_observation if self.counts else None

    def levels(self):
        return self.v.levels()

    def dump_nodes(self):
        return self.v.dump_nodes()

    def cull(self, pose):
        return self.v.frustum_cull(pose)[0]

    def render(self, pose, ds, colored):
        return self.v.render(pose, ds, colored=True) if colored else (self.v.render(pose, ds), None)

    def mesh(self, wmin, cm):
        return self.v.mesh(wmin, cm)


class EmuAdapter(OracleAdapter):
    """the host emulation of the engine's device code (tests/emu)"""

    def __init__(self, case: Case, pool_log2=17):
        from tests.emu.emu_py import EmuVolume
        self.v = EmuVolume(**case.config(), pool_log2=pool_log2)
        self.v.reset()

    def n_updates(self):
        return self.v.stats()["n_updates"]


# ---- exact ties (case T1) --------------------------------------------------------------------------------------------------
def tie_counts(case: Case, nodes):
    """For the stored nodes and every frame of `case`, count in float64 (exact here: every operand is dyadic):
    node centres whose projection u = x fx / z + cx or v = y fy / z + cy is exactly an integer, projections in (-1, 0),
    cloud points that lie on a node plane of the finest level, and observations d_new = z_pixel - z_node that equal
    0 or +-max_dist exactly."""
    cam, p = case.cam, case.params
    lv = nodes["keys"][:, 0].astype(np.int64)
    ijk = nodes["keys"][:, 1:].astype(np.float64)
    ctr = -case.size / 2 + (ijk + 0.5) * (case.size / np.exp2(lv))[:, None]
    vs = case.size / case.res
    n = dict(integer_proj=0, proj_in_minus1_0=0, points_on_planes=0, d_new_at_limits=0)
    lo, hi = p.get("min_sensor_dist", 0.3), p.get("max_sensor_dist", 3.0)
    for pose, cloud in case.frames():
        inv = np.linalg.inv(pose)
        assert np.array_equal(inv[:3, :3], pose[:3, :3].T)                     # (the inverse is exact)
        pc = ctr @ inv[:3, :3].T + inv[:3, 3]
        z = pc[:, 2]
        ok = (z >= lo) & (z <= hi)
        u = pc[ok, 0] * cam.fx / z[ok] + cam.cx
        v = pc[ok, 1] * cam.fy / z[ok] + cam.cy
        inimg = (u > -1) & (u < cam.width) & (v > -1) & (v < cam.height)
        n["integer_proj"] += int((inimg & ((u == np.round(u)) | (v == np.round(v)))).sum())
        n["proj_in_minus1_0"] += int((inimg & (((u > -1) & (u < 0)) | ((v > -1) & (v < 0)))).sum())
        pts = cloud[..., :3].reshape(-1, 3).astype(np.float64)
        pts = pts[np.isfinite(pts[:, 2])]
        w = pts @ pose[:3, :3].T + pose[:3, 3]
        on = np.any((w + case.size / 2) / vs == np.round((w + case.size / 2) / vs), axis=1)
        n["points_on_planes"] += int(on.sum())
        ui, vi = np.trunc(u).astype(np.int64), np.trunc(v).astype(np.int64)
        px = (ui >= 0) & (ui < cam.width) & (vi >= 0) & (vi < cam.height)
        zp = cloud[vi[px], ui[px], 2].astype(np.float64)
        dn = (zp - z[ok][px])[np.isfinite(zp)]
        pos, neg = p["max_dist_pos"], p["max_dist_neg"]
        n["d_new_at_limits"] += int(((dn == 0) | (dn == pos) | (dn == -neg)).sum())
    return n
