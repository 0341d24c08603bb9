"""Engine core (tsdf_core.cuh compiled for the host, tests/emu) vs the CPU oracle.

These run without a GPU.  They exercise exactly the code the CUDA kernels call — flat brick
layout, hash directory, per-node arithmetic, ray-march, marching cubes — and require results
that are bit-identical to the oracle at every node of every octree level (parity tier 3,
SURVEY.md §8a)."""
import numpy as np
import pytest

from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, assert_same_nodes, canon_soup, frames, query_points
from tests.emu.emu_py import EmuVolume


def pair(cfg, **kw):
    o = OracleVolume(**cfg, **{k: v for k, v in kw.items() if k not in ("track_variance", "pool_log2", "shard_rank", "shard_count")})
    e = EmuVolume(**cfg, **kw)
    o.reset(); e.reset()
    return o, e


def test_single_frame_256_exact():
    o, e = pair(CFG_256)
    pose = synth.orbit_pose(synth.S1, 0, 1)
    cloud = synth.make_frame(synth.S1, pose, CAM)
    o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())
    assert e.stats()["n_updates"] == o.stats().n_add_observation == 175900
    assert e.stats()["n_visits"] == o.stats().n_node_visits


def test_multi_frame_noise_color_variance_256():
    o, e = pair(CFG_256, integrate_color=1, track_variance=1)
    for pose, cloud in frames(synth.S1, 6, stride=9, color=True, noise_seed=11, dropout=0.02):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
        assert e.stats()["n_updates"] == o.stats().n_add_observation
    assert_same_nodes(o.dump_nodes(), e.dump_nodes(), rgb=True, var=True)


def test_orbit_512_prune_and_resplit():
    # a wide orbit makes earlier free-space observations prune and re-split (SURVEY.md §A.13-14)
    o, e = pair(CFG_512, pool_log2=17)
    for pose, cloud in frames(synth.S1, 5, stride=13, noise_seed=2):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())


def test_interior_2048_two_tiers():
    o, e = pair(CFG_2048, pool_log2=17)
    assert e.levels() == (5, 11, 2, 5)
    for pose, cloud in frames(synth.S2, 2, stride=3, noise_seed=4):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())


@pytest.mark.parametrize("res,size,cell", [(128, 3.0, 0.5), (1024, 3.0, 0.5), (256, 2.7, 0.3), (512, 12.0, 0.5)])
def test_other_tier_shapes(res, size, cell):
    # L-C = 4, 7, 5 ...: partial top tiers, permanently-split levels above the coarse depth, and a
    # grid size (2.7f) whose node centres are not exactly representable
    cfg = dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy,
               max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)
    o, e = pair(cfg, pool_log2=17)
    scene = synth.Scene(room_half=min(1.3, size * 0.45), cam_radius=0.8)
    for pose, cloud in frames(scene, 2, stride=6, noise_seed=9):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())
    pts = query_points(n=600)
    for mode in (0, 1):
        a, b = o.query(pts, 7, mode), e.query(pts, 7, mode)
        assert np.array_equal(a[3], b[3])
        for k in range(3):
            assert np.array_equal(a[k][a[3]], b[k][b[3]])
    # the mesh's brick walk, triangle for triangle in the reference's order (w_min 0: two frames leave weights of at most 2)
    va, _ = o.mesh(0.0, 0); vb, _ = e.mesh(0.0, 0)
    assert len(va) == len(vb) > 0
    assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).view(np.uint32))


def test_edge_cases_empty_nan_and_out_of_volume():
    o, e = pair(CFG_256)
    pose = synth.orbit_pose(synth.S1, 0, 1)
    empty = np.full((CAM.height, CAM.width, 4), np.nan, np.float32)
    o.integrate(empty, pose); e.integrate(empty, pose)           # all-NaN frame: nothing observed
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())
    assert o.stats().n_add_observation == e.stats()["n_updates"] == 0
    big = synth.Scene(room_half=4.0, cam_radius=1.0)                 # surface far outside the 3 m volume
    cloud = synth.make_frame(big, pose, CAM)
    o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())
    outside = np.eye(4); outside[:3, 3] = (5.0, 0.0, 0.0)           # camera outside the volume
    cloud = synth.make_frame(synth.S1, outside, CAM)
    o.integrate(cloud, outside); e.integrate(cloud, outside)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())


def test_frustum_cull_mask():
    o, e = pair(CFG_2048, pool_log2=12)
    for f in (0, 17, 33, 71):
        for scene in (synth.S1, synth.S2):
            pose = synth.orbit_pose(scene, f, 100)
            ma, ka = o.frustum_cull(pose); mb, kb = e.frustum_cull(pose)
            assert ka == kb and np.array_equal(ma, mb)


def test_queries_render_mesh_256():
    o, e = pair(CFG_256, integrate_color=1)
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    pts = query_points()
    for mode in (0, 1):
        a, b = o.query(pts, 7, mode), e.query(pts, 7, mode)
        assert np.array_equal(a[3], b[3]) and a[3].sum() > 1000
        for k in range(3):
            assert np.array_equal(a[k][a[3]].view(np.uint32), b[k][b[3]].view(np.uint32))
    pose = synth.orbit_pose(synth.S1, 10, 100)
    ra, ca = o.render(pose, 4, colored=True)
    rb, cb = e.render(pose, 4, colored=True)
    assert np.isfinite(ra[..., 2]).sum() > 5000
    assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True)       # per-pixel depth: exact (bar: 1e-4 m)
    assert np.array_equal(ra[..., 4:7], rb[..., 4:7], equal_nan=True)
    assert np.array_equal(ca, cb)
    for cm, wmin in ((0, 2.0), (1, 0.0), (2, 2.5)):
        va, cola = o.mesh(wmin, cm); vb, colb = e.mesh(wmin, cm)
        assert len(va) == len(vb) > 3000
        assert np.array_equal(canon_soup(va, cola), canon_soup(vb, colb))
        # and in the reference's own triangle order (depth-first over the octree): the engine sorts by mc_order_key
        assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).view(np.uint32))
        assert cola is None or np.array_equal(cola, colb)


def test_global_transform_applies_to_mesh_only():
    gt = np.eye(4); gt[:3, 3] = (0.25, -1.0, 2.0); gt[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    o, e = pair(CFG_256, global_transform=gt)
    for pose, cloud in frames(synth.S1, 2, stride=5):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes())
    va, _ = o.mesh(1.0, 0); vb, _ = e.mesh(1.0, 0)
    assert len(va) > 1000 and np.array_equal(canon_soup(va), canon_soup(vb))


@pytest.mark.parametrize("cap", ["0", "16", "128"])
def test_breadth_first_fresh_subtree_visit_equals_the_recursion(cap, monkeypatch):
    """fresh_children_bfs (the cooperative re-split visit of k_celltop_up) driven by one emulated lane for EVERY split of
    the frame: record capacity 128, 16 (most subtrees overflow into the depth-first fallback) and 0 (recursion only)."""
    monkeypatch.setenv("B2_EMU_BFS_CAP", cap)
    o, e = pair(CFG_256, integrate_color=1)
    for pose, cloud in frames(synth.S1, 6, stride=9, color=True, noise_seed=11):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert_same_nodes(o.dump_nodes(), e.dump_nodes(), rgb=True)
    so, se = o.stats(), e.stats()
    assert so.n_add_observation == se["n_updates"] and so.n_node_visits == se["n_visits"]
    monkeypatch.setenv("B2_EMU_BFS_CAP", "128")
