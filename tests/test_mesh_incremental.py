"""Incremental meshing on the host emulation of the engine's device code (tests/emu): the change epochs per coarse cell that
k_front, presplit_point and k_edit_store stamp, and marching cubes restricted to a set of cells (DESIGN.md §3g).

For every pair of consecutive epochs of each stream, at w_min 0 and 2 and colour by RGB and by confidence:
* every cell whose triangle run differs between the two full meshes is in the mask b200tsdf_changed_cells reports;
* re-meshing the masked cells and splicing their runs into the earlier mesh gives the later full mesh, bit for bit;
* the mesh of random cell sets (none, all, single cells on the grid border) is the full mesh's runs of those cells.
A constructed stream checks that a frame's pre-split of points beyond max_sensor_dist, in cells it does not cull in, is
reported."""
import numpy as np
import pytest

from cpu_tsdf_b200 import synth
from tests import edit_cases
from tests.common import CFG_256, frames
from tests.dynamic_cases import CASES
from tests.emu import cells_py
from tests.emu.cells_py import CellsEmuVolume
from tests.general_cases import look_at_pose

MODES = [(0.0, 1), (2.0, 1), (0.0, 2), (2.0, 2)]


def border_cells(n, rng, k=6):
    """k cells on the faces, edges and corners of the n^3 grid of coarse cells"""
    out = [0, n * n * n - 1, (n - 1) * n * n, n - 1]
    while len(out) < k:
        x, y, z = rng.integers(0, n, 3)
        x = rng.choice([0, n - 1])
        out.append(int((x * n + y) * n + z))
    return out


class Tracker:
    """the full meshes of the last epoch, per (w_min, colour mode), and the checks against the next epoch"""

    def __init__(self, vol, seed=0, modes=MODES):
        self.vol = vol
        self.modes = modes
        self.rng = np.random.default_rng(seed)
        self.prev = None
        self.steps = 0
        self.changed_cells = 0

    def snapshot(self):
        return {m: cells_py.mesh_cells(self.vol, *m) for m in self.modes}

    def step(self):
        now, _ = cells_py.changed_cells(self.vol, 0)
        meshes = self.snapshot()
        if self.prev is not None:
            since, old = self.prev
            assert now > since, "a mutation did not advance the epoch"
            _, mask = cells_py.changed_cells(self.vol, since)
            for m in self.modes:
                ov, oc, ocnt = old[m]
                nv, nc, ncnt = meshes[m]
                # every cell whose run changed is reported
                orun, nrun = cells_py.runs(ov, ocnt), cells_py.runs(nv, ncnt)
                diff = [c for c in range(len(mask)) if ocnt[c] != ncnt[c] or not np.array_equal(orun[c].view(np.uint32), nrun[c].view(np.uint32))]
                missed = [c for c in diff if not mask[c]]
                assert not missed, f"mode {m}: cells {missed[:10]} changed but are not in the mask"
                self.changed_cells += len(diff)
                # re-mesh the masked cells and splice them into the earlier mesh
                sv, sc, scnt = cells_py.mesh_cells(self.vol, *m, mask)
                assert np.array_equal(scnt[mask == 0], np.zeros(int((mask == 0).sum()), np.int64))
                assert np.array_equal(scnt[mask != 0], ncnt[mask != 0])
                got, counts = cells_py.splice(ov, ocnt, sv, scnt, mask)
                assert np.array_equal(counts, ncnt)
                assert np.array_equal(got.view(np.uint32), nv.view(np.uint32)), f"mode {m}: spliced mesh differs from the full mesh"
                if nc is not None:
                    gc, _ = cells_py.splice(oc, ocnt, sc, scnt, mask)
                    assert np.array_equal(gc, nc)
        if self.steps % 2 == 0:
            self.random_masks(meshes)
        self.prev = (now, meshes)
        self.steps += 1

    def random_masks(self, meshes):
        m = self.modes[(self.steps // 2) % len(self.modes)]
        fv, fc, fcnt = meshes[m]
        ncells = len(fcnt)
        n = round(ncells ** (1 / 3))
        perm = cells_py.morton_cells(ncells)
        cell_of = np.repeat(perm, fcnt[perm])                    # the cell of each vertex: cells follow in Morton order
        masks = [np.zeros(ncells, np.uint8), np.ones(ncells, np.uint8)]
        for c in border_cells(n, self.rng):
            mk = np.zeros(ncells, np.uint8); mk[c] = 1; masks.append(mk)
        masks.append((self.rng.random(ncells) < 0.2).astype(np.uint8))
        for mk in masks:
            v, c, cnt = cells_py.mesh_cells(self.vol, *m, mk)
            keep = mk[cell_of] != 0
            assert np.array_equal(v.view(np.uint32), fv[keep].view(np.uint32))
            if fc is not None:
                assert np.array_equal(c, fc[keep])
            assert np.array_equal(cnt, np.where(mk != 0, fcnt, 0))


def test_rgb_stream_256():
    vol = CellsEmuVolume(**CFG_256, integrate_color=1, pool_log2=16)
    vol.reset()
    t = Tracker(vol, 1)
    t.step()
    for pose, cloud in frames(synth.S1, 6, stride=9, color=True, noise_seed=3):
        vol.integrate(cloud, pose)
        t.step()
    assert t.changed_cells > 0


@pytest.mark.parametrize("cid", ["K1", "K2", "K6"])
def test_dynamic_cases(cid):
    case = CASES[cid]
    vol = CellsEmuVolume(**case.config(), track_variance=int(case.track_variance), pool_log2=17)
    vol.reset()
    t = Tracker(vol, 2, MODES if case.res <= 256 else MODES[::3])     # 512^3: (w_min 0, RGB) and (w_min 2, confidence)
    t.step()
    for pose, cloud in case.frames():
        vol.integrate(cloud, pose)
        t.step()
    assert t.changed_cells > 0


class EditAdapter:
    def __init__(self, sc, tracker_seed):
        self.v = CellsEmuVolume(**sc.config(), track_variance=int(sc.track_variance), pool_log2=17)
        self.v.reset()
        self.t = Tracker(self.v, tracker_seed, MODES if sc.cfg["xres"] <= 256 else MODES[::3])
        self.t.step()

    def integrate(self, cloud, pose):
        self.v.integrate(cloud, pose)
        self.t.step()

    def levels(self):
        return self.v.levels()

    def write(self, pts, d, w, ms):
        before, _ = cells_py.changed_cells(self.v, 0)
        st = self.v.set_containing_voxels(pts, d, w, ms)
        after, _ = cells_py.changed_cells(self.v, 0)
        assert after == before + int((st == 0).any()), "a write batch advances the epoch by one iff it writes a node"
        if after != before:
            self.t.step()
        return st


@pytest.mark.parametrize("sid", ["sphere_256_rgb", "carve_512"])
def test_edit_scenarios(sid):
    sc = edit_cases.SCENARIOS[sid]
    a = EditAdapter(sc, 3)
    edit_cases.run(sc, a)
    assert a.t.changed_cells > 0


def nodes_per_cell(vol):
    d = vol.dump_nodes()
    C = vol.levels()[0]
    k = d["keys"][d["keys"][:, 0] >= C]
    sh = k[:, 0] - C
    n = 1 << C
    cell = ((k[:, 1] >> sh) * n + (k[:, 2] >> sh)) * n + (k[:, 3] >> sh)
    return np.bincount(cell, minlength=n ** 3)


def test_presplit_beyond_far_plane_is_reported():
    """a surface seen from near, then a frame whose every point lies beyond max_sensor_dist: its pre-split adds nodes in cells
    that it does not cull in (no update reaches them), and the mask reports every such cell and every cell whose mesh changed"""
    cfg = dict(CFG_256, integrate_color=1, max_sensor_dist=0.7, pool_log2=16)
    vol = CellsEmuVolume(**cfg)
    vol.reset()
    cam = synth.Camera()
    near = look_at_pose((0.9, 0.05, 0.02), (0.0, 0.0, 0.0))
    far = look_at_pose((1.32, -0.03, 0.04), (0.0, 0.0, 0.0))
    f0 = synth.make_frame(synth.S1, near, cam, color=True, noise_seed=5, frame=0)
    vol.integrate(f0, near)
    since, _ = cells_py.changed_cells(vol, 0)
    v0, _, c0 = cells_py.mesh_cells(vol, 0.0, 1)
    n0 = nodes_per_cell(vol)
    cull, _ = vol.frustum_cull(far)
    # the far frame: the near frame's points moved 6 cm towards the cameras, in front of the surface; every one of them lies
    # beyond max_sensor_dist from the far camera
    p = f0[..., :3].astype(np.float64)
    p = p - 0.06 * p / np.linalg.norm(p, axis=-1, keepdims=True)
    world = p @ near[:3, :3].T + near[:3, 3]
    inv = np.linalg.inv(far)
    f1 = f0.copy()
    f1[..., :3] = (world @ inv[:3, :3].T + inv[:3, 3]).astype(np.float32)
    ok = ~np.isnan(f1[..., 2])
    assert np.all(np.linalg.norm(f1[..., :3][ok], axis=-1) > 0.7)
    vol.integrate(f1, far)
    v1, _, c1 = cells_py.mesh_cells(vol, 0.0, 1)
    n1 = nodes_per_cell(vol)
    _, mask = cells_py.changed_cells(vol, since)
    culled = cull.reshape(-1) != 0
    split_outside = np.flatnonzero((n1 > n0) & ~culled)
    assert len(split_outside), "the far frame split no node outside its cull list"
    assert mask[split_outside].all()
    r0, r1 = cells_py.runs(v0, c0), cells_py.runs(v1, c1)
    changed = [c for c in range(len(c0)) if c0[c] != c1[c] or not np.array_equal(r0[c], r1[c])]
    assert all(mask[c] for c in changed)
