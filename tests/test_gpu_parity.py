"""CUDA engine (through the C ABI / Python mirror) vs the CPU oracle on a real H100.

Bar (north_star): per-voxel {sdf,weight} and mesh vertices within a stated float tolerance,
renderView depth within 1e-4 m.  The engine reproduces the reference's arithmetic expression by
expression, so the tests demand BIT-EXACT equality at every node of every octree level, on every
render pixel and on every mesh vertex; the tolerances of the north star are upper bounds."""
import os

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, assert_same_nodes, canon_soup, frames, query_points

pytestmark = pytest.mark.gpu


def make_engine(cfg, pool_log2=17, **kw):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, track_variance=bool(kw.pop("track_variance", 0)))
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg.get("xsize", 3.0), cfg.get("ysize", 3.0), cfg.get("zsize", 3.0))
    v.setCameraIntrinsics(cfg.get("fx", 525.0), cfg.get("fy", 525.0), cfg["cx"], cfg["cy"])
    if "max_cell_x" in cfg:
        v.setMaxVoxelSize(cfg["max_cell_x"], cfg["max_cell_y"], cfg["max_cell_z"])
    if kw.get("integrate_color"):
        v.setIntegrateColor(True)
    if "max_weight" in kw:
        v.setWeightTruncationLimit(kw["max_weight"])
    if "global_transform" in kw:
        v.setGlobalTransform(kw["global_transform"])
    v.reset()
    return v


def pair(cfg, pool_log2=17, **kw):
    o = OracleVolume(**cfg, **{k: v for k, v in kw.items() if k != "track_variance"})
    o.reset()
    return o, make_engine(cfg, pool_log2, **kw)


def test_engine_library_is_the_cuda_one(engine_lib):
    # the path under test is the in-tree CUDA library; nothing else implements the ABI
    assert os.path.samefile(engine_lib, pkg.LIB_PATH)
    maps = open("/proc/self/maps").read()
    make_engine(CFG_256, 12)
    assert "libb200tsdf.so" in open("/proc/self/maps").read() or "libb200tsdf.so" in maps


def test_single_frame_256_exact():
    o, e = pair(CFG_256)
    pose = synth.orbit_pose(synth.S1, 0, 1)
    cloud = synth.make_frame(synth.S1, pose, CAM)
    o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())
    st = e.stats()
    assert st.n_updates == o.stats().n_add_observation == 175900
    assert st.n_culled_cells == o.stats().n_culled_cells


def test_multi_frame_noise_color_variance_256():
    o, e = pair(CFG_256, integrate_color=1, track_variance=1)
    for pose, cloud in frames(synth.S1, 6, stride=9, color=True, noise_seed=11, dropout=0.02):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
        assert e.stats().n_updates == o.stats().n_add_observation
    assert_same_nodes(o.dump_nodes(), e.download_nodes(), rgb=True, var=True)


def test_orbit_512_config2():
    o, e = pair(CFG_512, 18)
    for pose, cloud in frames(synth.S1, 10, stride=10, noise_seed=2):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())
    for f in (0, 25, 50, 75):
        pose = synth.orbit_pose(synth.S1, f, 100)
        ra = o.render(pose, 2); rb = e.renderView(pose, 2)
        good = np.isfinite(ra[..., 2])
        assert good.sum() > 20000
        assert np.array_equal(np.isfinite(rb[..., 2]), good)
        assert np.nanmax(np.abs(ra[..., 2] - rb[..., 2])) <= 1e-4        # north-star bar
        assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True)   # what we actually hold
        assert np.array_equal(ra[..., 4:7], rb[..., 4:7], equal_nan=True)


def test_interior_2048_config3_color_mesh():
    o, e = pair(CFG_2048, 18, integrate_color=1)
    for pose, cloud in frames(synth.S2, 4, stride=2, color=True, noise_seed=4):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
        assert e.stats().n_updates == o.stats().n_add_observation
    assert_same_nodes(o.dump_nodes(), e.download_nodes(), rgb=True)
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(e)
    for wmin, rgb in ((2.0, True), (0.0, False)):
        mc.setMinWeight(wmin); mc.setColorByRGB(rgb)
        vb, cb, polys = mc.reconstruct()
        va, ca = o.mesh(wmin, 1 if rgb else 0)
        assert len(va) == len(vb) > 10000 and len(polys) * 3 == len(vb)
        assert np.array_equal(canon_soup(va, ca), canon_soup(vb, cb))
        # and triangle for triangle in the reference's own order (the engine sorts its emission by mc_order_key)
        assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).reshape(-1, 3).view(np.uint32)) and (ca is None or np.array_equal(ca, cb))
        assert np.abs(canon_soup(va)[:, :9] - canon_soup(vb)[:, :9]).max() <= 1e-5   # north-star bar


@pytest.mark.parametrize("res,size,cell", [(128, 3.0, 0.5), (1024, 3.0, 0.5), (256, 2.7, 0.3), (512, 12.0, 0.5)])
def test_other_tier_shapes(res, size, cell):
    cfg = dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy,
               max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)
    o, e = pair(cfg)
    scene = synth.Scene(room_half=min(1.3, size * 0.45), cam_radius=0.8)
    for pose, cloud in frames(scene, 2, stride=6, noise_seed=9):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())
    # the mesh's brick walk, triangle for triangle in the reference's order (w_min 0: two frames leave weights of at most 2)
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(e)
    mc.setMinWeight(0.0)
    vb, _, _ = mc.reconstruct()
    va, _ = o.mesh(0.0, 0)
    assert len(va) == len(vb) > 0
    assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).reshape(-1, 3).view(np.uint32))


def test_edge_cases_empty_nan_and_out_of_volume():
    o, e = pair(CFG_256)
    pose = synth.orbit_pose(synth.S1, 0, 1)
    empty = np.full((CAM.height, CAM.width, 4), np.nan, np.float32)
    o.integrate(empty, pose); e.integrateCloud(empty, None, pose)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())
    assert e.stats().n_updates == 0
    big = synth.Scene(room_half=4.0, cam_radius=1.0)
    cloud = synth.make_frame(big, pose, CAM)
    o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    outside = np.eye(4); outside[:3, 3] = (5.0, 0.0, 0.0)
    cloud = synth.make_frame(synth.S1, outside, CAM)
    o.integrate(cloud, outside); e.integrateCloud(cloud, None, outside)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())


def test_weight_saturation_and_reset_idempotence():
    o, e = pair(CFG_256, max_weight=3)
    pose = synth.orbit_pose(synth.S1, 0, 1)
    cloud = synth.make_frame(synth.S1, pose, CAM, noise_seed=1)
    for _ in range(5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    a = e.download_nodes()
    assert_same_nodes(o.dump_nodes(), a)
    assert a["dw"][:, 1].max() == 3.0
    e.reset(); o.reset()
    b = e.download_nodes()
    assert len(b["keys"]) == 512 and (b["dw"] == [-1, 0]).all()
    o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    assert_same_nodes(o.dump_nodes(), e.download_nodes())


def test_frustum_cull_mask():
    o, e = pair(CFG_2048, 12)
    for f in (0, 17, 33, 71):
        for scene in (synth.S1, synth.S2):
            pose = synth.orbit_pose(scene, f, 100)
            ma, ka = o.frustum_cull(pose)
            mb = e.getFrustumCulledVoxels(pose)
            assert ka == mb.sum() and np.array_equal(ma.astype(bool), mb)


def test_queries_render_mesh_256():
    o, e = pair(CFG_256, integrate_color=1)
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    pts = query_points()
    for mode, fn in ((0, None), (1, None)):
        a = o.query(pts, 7, mode)
        b = e._query(pts, 7, mode)
        assert np.array_equal(a[3], b[3]) and a[3].sum() > 1000
        for k in range(3):
            assert np.array_equal(a[k][a[3]].view(np.uint32), b[k][b[3]].view(np.uint32))
    ok, val = e.getFxn(pts[0])
    assert isinstance(ok, bool)
    pose = synth.orbit_pose(synth.S1, 10, 100)
    ra, ca = o.render(pose, 1, colored=True)
    rb, cb = e.renderColoredView(pose, 1)
    assert np.isfinite(ra[..., 2]).sum() > 100000
    assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True)
    assert np.array_equal(ra[..., 4:7], rb[..., 4:7], equal_nan=True)
    assert np.array_equal(ca, cb)
    mc = pkg.MarchingCubesTSDFOctree(); mc.setInputTSDF(e)
    for cm, wmin in ((0, 2.0), (1, 0.0), (2, 2.5)):
        mc.setMinWeight(wmin); mc.setColorByRGB(cm == 1); mc.setColorByConfidence(cm == 2)
        vb, colb, _ = mc.reconstruct()
        va, cola = o.mesh(wmin, cm)
        assert len(va) == len(vb) > 3000
        assert np.array_equal(canon_soup(va, cola), canon_soup(vb, colb))
        assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).reshape(-1, 3).view(np.uint32)) and (cola is None or np.array_equal(cola, colb))


def test_save_vol_matches_oracle_bytes(tmp_path):
    o, e = pair(CFG_256, integrate_color=1, track_variance=1)
    for pose, cloud in frames(synth.S1, 3, stride=7, color=True, noise_seed=5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    pa, pb = str(tmp_path / "a.vol"), str(tmp_path / "b.vol")
    assert o.save(pa) == 0
    e.save(pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()


def test_errors_are_reported_not_thrown():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    with pytest.raises(pkg.B200Error):
        v.integrateCloud(np.zeros((4, 4, 4), np.float32), None, np.eye(4))     # before reset()
    v.setResolution(100, 100, 100)
    with pytest.raises(pkg.B200Error):
        v.reset()                                                              # not a power of two
    v.setResolution(256, 256, 256); v.reset()
    with pytest.raises(pkg.B200Error):
        v.integrateCloud(np.zeros((4, 4, 4), np.float32), None, np.eye(4))     # cloud is not image-sized
    # repeated single-point queries reuse the handle's scratch (no allocation per call) and stay consistent
    pose0 = synth.orbit_pose(synth.S1, 0, 1)
    v.setCameraIntrinsics(525, 525, CAM.cx, CAM.cy)
    v.integrateCloud(synth.make_frame(synth.S1, pose0, CAM), None, pose0)
    pts = query_points(seed=5, n=64)
    bval, _, _, bok = v._query(pts, 7, 1)
    for i in range(0, 64, 7):
        val, _, _, ok = v._query(pts[i:i + 1], 7, 1)
        assert ok[0] == bok[i] and np.array_equal(val.view(np.uint32), bval[i:i + 1].view(np.uint32))
    # a pool that is too small must surface as ENOMEM, not corrupt memory
    small = pkg.TSDFVolumeOctree(device=0, pool_log2=8)
    small.setResolution(512, 512, 512); small.setCameraIntrinsics(525, 525, CAM.cx, CAM.cy); small.reset()
    pose = synth.orbit_pose(synth.S1, 0, 1)
    with pytest.raises(pkg.B200Error):
        small.integrateCloud(synth.make_frame(synth.S1, pose, CAM), None, pose)
        small.sync()


def test_sharded_volumes_union_is_the_whole_volume():
    # DESIGN.md §5: shard by coarse cell; here both shards live on one GPU (two handles), the multi-GPU
    # launch in bench.py only changes the device ordinal
    from tests.shard_worker import cell_owner
    o = OracleVolume(**CFG_256); o.reset()
    shards = []
    for r in range(2):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=16, shard_rank=r, shard_count=2)
        v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy); v.reset()
        shards.append(v)
    total = 0
    for pose, cloud in frames(synth.S1, 3, stride=11, noise_seed=21):
        o.integrate(cloud, pose); total += o.stats().n_add_observation
        for v in shards:
            v.integrateCloud(cloud, None, pose)
            total -= v.stats().n_updates
    assert total == 0                                     # every voxel update happened on exactly one shard
    ref = o.dump_nodes()
    C = o.levels()[0]
    owner = np.array([cell_owner(*c, 2) for c in (ref["keys"][:, 1:] >> (ref["keys"][:, 0:1] - C))])
    for r, v in enumerate(shards):
        d = v.download_nodes()
        own = np.array([cell_owner(*c, 2) for c in (d["keys"][:, 1:] >> (d["keys"][:, 0:1] - C))]) == r
        assert np.array_equal(d["keys"][own], ref["keys"][owner == r])
        assert np.array_equal(d["dw"][own].view(np.uint32), ref["dw"][owner == r].view(np.uint32))
        assert (d["dw"][~own] == [-1, 0]).all() and not d["split"][~own].any()


def test_load_vol_written_by_the_reference_path(tmp_path):
    # TSDFVolumeOctree::load (cpp:248-275): import a .vol written by the oracle, continue fusing, and stay exact
    o, e = pair(CFG_256, integrate_color=1, track_variance=1)
    fr = list(frames(synth.S1, 4, stride=7, color=True, noise_seed=5))
    for pose, cloud in fr[:2]:
        o.integrate(cloud, pose)
    pa = str(tmp_path / "a.vol")
    assert o.save(pa) == 0
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=17, track_variance=True)
    v.load(pa)
    assert v.getResolution() == (256, 256, 256) and v.getCameraIntrinsics()[2] == CAM.cx
    assert_same_nodes(o.dump_nodes(), v.download_nodes(), rgb=True, var=True)
    for pose, cloud in fr[2:]:
        o.integrate(cloud, pose); v.integrateCloud(cloud, None, pose)
    assert_same_nodes(o.dump_nodes(), v.download_nodes(), rgb=True, var=True)
    pb = str(tmp_path / "b.vol")
    v.save(pb); o.save(pa)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    with pytest.raises(pkg.B200Error):
        v.load(str(tmp_path / "missing.vol"))
    # a header that switches weight_by_depth_ on (cpp:240, 265; hpp:200-201) is refused, not silently fused with w_new = 1
    raw = open(pa, "rb").read()
    head, tail = raw.split(b"% 4 4", 1)
    lines = head.split(b"\n")
    assert lines[-3:-1] == [b"0", b"0"]                       # weight_by_depth_, weight_by_variance_ (the last header lines before the transform)
    lines[-3] = b"1"
    pc = str(tmp_path / "c.vol")
    open(pc, "wb").write(b"\n".join(lines) + b"% 4 4" + tail)
    with pytest.raises(pkg.B200Error, match="weight_by"):
        v.load(pc)


def _engine_2048(general=False, pool_log2=18):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy); v.setIntegrateColor(True)
    if general:
        v._cfg.debug_flags = 1            # debug switch: general depth-first update kernel only
        v._push()
    v.reset()
    return v


def test_full_size_stream_properties_2048(tmp_path):
    # BASELINE.json's full size (640x480 into 2048^3, colour).  The 100-frame stream is compared with the reference itself in
    # tests/test_golden.py (digests from oracle/_ref: nodes at 50 / 100 frames, renderView, marching cubes at w_min 2 and 0);
    # here a 40-frame stream is checked through size-independent properties: stored values stay in the reference's ranges,
    # save -> load -> save is the identity on bytes, and the reloaded volume renders identically.
    fast = _engine_2048(False)
    upd = 0
    for f in range(40):
        pose = synth.orbit_pose(synth.S2, f, 100)
        cloud = synth.make_frame(synth.S2, pose, CAM, color=True, noise_seed=77, frame=f)
        fast.integrateCloud(cloud, None, pose)
        if f % 13 == 0:
            upd += fast.stats().n_updates
    assert upd > 1_000_000
    a = fast.download_nodes()
    assert len(a["keys"]) > 2_000_000
    d, w = a["dw"][:, 0], a["dw"][:, 1]
    assert w.min() >= 0 and w.max() <= 100.0 and d.min() >= -1.0 and d.max() <= 1.0       # octree.cpp:156-159, hpp:189-198
    assert ((w == 0) <= (d == -1.0)).all()                                                  # never-observed nodes keep the constructor state
    lv = a["keys"][:, 0]
    assert lv.min() == 5 and lv.max() == 11 and not a["split"][lv == 11].any()
    pa, pb = str(tmp_path / "a.vol"), str(tmp_path / "b.vol")
    fast.save(pa)
    again = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
    again.load(pa); again.save(pb)
    import hashlib
    ha = hashlib.sha256(open(pa, "rb").read()).hexdigest(); hb = hashlib.sha256(open(pb, "rb").read()).hexdigest()
    assert ha == hb
    # and the render of the reloaded volume is identical
    pose = synth.orbit_pose(synth.S2, 20, 100)
    assert np.array_equal(fast.renderView(pose, 4), again.renderView(pose, 4), equal_nan=True)   # (same wrapper on both sides)


def test_4096_three_tiers_config5_shape():
    # BASELINE.json configs[4] grid: 4096^3 over 10 m (L=12, C=5, three tiers, coarse cells inside the top bricks)
    cfg = dict(xres=4096, yres=4096, zres=4096, xsize=10.0, ysize=10.0, zsize=10.0, cx=CAM.cx, cy=CAM.cy)
    o, e = pair(cfg, 19)
    assert e.stats().tiers == 3
    for pose, cloud in frames(synth.S2, 2, stride=3, noise_seed=4):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
        assert e.stats().n_updates == o.stats().n_add_observation
    assert_same_nodes(o.dump_nodes(), e.download_nodes())


def test_4096_batches_replay_graphs_with_the_coarse_sweeps():
    """Shapes with coarse levels above the tier-1 supercells (4096^3 / 10 m: one such level) launch k_upper_down / k_upper_up
    around the four fused kernels; these read the frame from its record too, so a batch is one captured graph.  Two batches
    (3 + 3 frames: capture, then replay on the other half of the record ring) against the oracle frame by frame."""
    import torch
    cfg = dict(xres=4096, yres=4096, zres=4096, xsize=10.0, ysize=10.0, zsize=10.0, cx=CAM.cx, cy=CAM.cy)
    o, e = pair(cfg, 19)
    fs = list(frames(synth.S2, 6, stride=3, noise_seed=8))
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fs]
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    H, W = fs[0][1].shape[:2]
    e.profile_begin()
    for lo, hi in ((0, 3), (3, 6)):
        e.integrateBatchDevice([d.data_ptr() for d in dev[lo:hi]], H, W, 4 * fs[0][1].shape[2], [p for p, _ in fs[lo:hi]])
    prof = e.profile_end()
    assert prof.graph_launches == 2
    assert_same_nodes(o.dump_nodes(), e.download_nodes())
    assert e.stats().n_updates == o.stats().n_add_observation


def test_shards_gathered_into_one_volume_render_like_the_whole():
    # multi-GPU read side (SURVEY.md §8e): integrate in shards, gather the shards into one volume, render / mesh there
    o = OracleVolume(**CFG_512); o.reset()
    shards = []
    for r in range(3):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=17, shard_rank=r, shard_count=3)
        v.setResolution(512, 512, 512); v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy); v.reset()
        shards.append(v)
    for pose, cloud in frames(synth.S1, 4, stride=11, noise_seed=21):
        o.integrate(cloud, pose)
        for v in shards:
            v.integrateCloud(cloud, None, pose)
    whole = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
    whole.setResolution(512, 512, 512); whole.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy); whole.reset()
    for v in shards:
        whole.import_shard(v.export_shard())
    assert_same_nodes(o.dump_nodes(), whole.download_nodes())
    pose = synth.orbit_pose(synth.S1, 17, 100)
    ra, rb = o.render(pose, 2), whole.renderView(pose, 2)
    assert np.isfinite(ra[..., 2]).sum() > 20000
    assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True) and np.array_equal(ra[..., 4:7], rb[..., 4:7], equal_nan=True)
    with pytest.raises(pkg.B200Error):
        other = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
        other.setResolution(256, 256, 256); other.reset()
        other.import_shard(shards[0].export_shard())          # different grid


def test_batch_graph_replay_matches_the_oracle_and_frame_by_frame():
    """b200tsdf_integrate_batch_device: the frames of a batch are replayed from one captured CUDA graph (records in a device
    ring).  Three batches (sizes 5, 5, 3: the second replays the first one's graph on the other half of the ring) must leave
    exactly the volume the oracle builds frame by frame."""
    import torch
    o, e = pair(CFG_512, 18, integrate_color=1)
    fs = list(frames(synth.S1, 13, stride=7, color=True, noise_seed=21))
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fs]
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    H, W = fs[0][1].shape[:2]
    for lo, hi in ((0, 5), (5, 10), (10, 13)):
        assert fs[0][1].shape[2] == 8                                  # pcl::PointXYZRGBA rows
        e.integrateBatchDevice([d.data_ptr() for d in dev[lo:hi]], H, W, 32, [p for p, _ in fs[lo:hi]], rgba_off=16)
    e.sync()
    assert_same_nodes(o.dump_nodes(), e.download_nodes(), rgb=True)
    assert e.stats().n_updates == o.stats().n_add_observation
    # a configuration fused by the general depth-first kernel (here: track_variance) takes the frame-by-frame route inside the same call
    o2, e2 = pair(CFG_256, 16, track_variance=1)
    fs2 = list(frames(synth.S1, 3, stride=9, noise_seed=5))
    dev2 = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fs2]
    for pose, cloud in fs2:
        o2.integrate(cloud, pose)
    e2.integrateBatchDevice([d.data_ptr() for d in dev2], H, W, 4 * fs2[0][1].shape[2], [p for p, _ in fs2])
    e2.sync()
    assert_same_nodes(o2.dump_nodes(), e2.download_nodes())


@pytest.mark.parametrize("host_pack", ["1", "0"])
def test_batch_rows_from_host_buffers_one_gpu(host_pack, monkeypatch):
    """b200tsdf_integrate_batch_rows on one GPU (the end-to-end path of bench.py): HOST rows in, packed to 16-byte pixels by
    the host thread pool (B200TSDF_HOST_PACK=1, the default; 3 threads here so the fork/join is exercised) or uploaded as
    they are (=0); either way the volume is the oracle's, bit for bit.  Batches of 9 and 4 frames: chunks of 8 + 1, then a
    short batch on the second buffer set, then the first set again."""
    monkeypatch.setenv("B200TSDF_HOST_PACK", host_pack)
    monkeypatch.setenv("B200TSDF_PACK_THREADS", "3")
    o, e = pair(CFG_512, 18, integrate_color=1)
    fs = list(frames(synth.S1, 17, stride=5, color=True, noise_seed=33))
    host = [np.ascontiguousarray(c) for _, c in fs]
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    H, W = host[0].shape[:2]
    assert e.rowSlice(H) == (0, H)
    for lo, hi in ((0, 9), (9, 13), (13, 17)):
        e.integrateBatchRows([c.ctypes.data for c in host[lo:hi]], H, W, 32, [p for p, _ in fs[lo:hi]], rgba_off=16)
    e.sync()
    assert_same_nodes(o.dump_nodes(), e.download_nodes(), rgb=True)
    assert e.stats().n_updates == o.stats().n_add_observation


def test_get_tsdf_value_direct_entry_point():
    """b200tsdf_interpolate = getTSDFValue / interpolateTrilinearly (cpp:454-541): value bits, NaN on the border layer and outside,
    and the in/out `valid` flag, against the oracle (itself pinned to the reference for this call in tests/test_ref_pin.py)."""
    from tests.test_ref_pin import _interp_points
    o, e = pair(CFG_256)
    for pose, cloud in frames(synth.S1, 3, stride=9, noise_seed=5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    pts = _interp_points()
    for vin in (True, False):
        va, oa = o.interpolate(pts, vin); vb, ob = e.getTSDFValue(pts, vin)
        assert np.array_equal(oa, ob)
        assert np.array_equal(np.isnan(va), np.isnan(vb))            # (the payload bits of a NaN are not part of the contract)
        fin = ~np.isnan(va)
        assert np.array_equal(va[fin].view(np.uint32), vb[fin].view(np.uint32))
    assert e.getTSDFValue(pts, True)[1].sum() > 500


def test_rgb_normalized_payload_in_the_engine(tmp_path):
    """setColorMode ("RGBNormalized") (tsdf_volume_octree.h:290; RGBNormalized::addObservation / getRGB / serialize, octree.cpp:379-434):
    the four floats of every node, the uint8 colours getRGB derives from them (renderColoredView, mesh colours) and the .vol bytes —
    against the restatement, which tests/test_ref_pin.py pins to the reference for exactly this payload."""
    o = OracleVolume(**CFG_256, integrate_color=1, color_mode=1); o.reset()
    e = pkg.TSDFVolumeOctree(device=0, pool_log2=17, track_variance=True)      # (M_ / nsample_ are part of the .vol bytes)
    e.setResolution(256, 256, 256); e.setGridSize(3.0, 3.0, 3.0); e.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy)
    e.setIntegrateColor(True); e.setColorMode("RGBNormalized"); e.reset()
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    da, db = o.dump_nodes(), e.download_nodes()
    assert_same_nodes(da, db, rgb=True)
    assert np.array_equal(da["rgbn"].view(np.uint32), db["rgbn"].view(np.uint32))          # NaNs of black pixels included, bit for bit
    assert (da["dw"][:, 1] > 0).sum() > 50000
    pose = synth.orbit_pose(synth.S1, 10, 100)
    ra, ca = o.render(pose, 4, colored=True); rb, cb = e.renderColoredView(pose, 4)
    assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True) and np.array_equal(ca, cb) and ca.any()
    mc = pkg.MarchingCubesTSDFOctree(); mc.setInputTSDF(e); mc.setMinWeight(0.0); mc.setColorByRGB(True)
    vb, colb, _ = mc.reconstruct()
    va, cola = o.mesh(0.0, 1)
    assert len(va) > 3000 and np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).reshape(-1, 3).view(np.uint32)) and np.array_equal(cola, colb)
    pa, pb = str(tmp_path / "a.vol"), str(tmp_path / "b.vol")
    assert o.save(pa) == 0
    e.save(pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    # LAB is refused loudly rather than silently fused as something else
    lab = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    lab.setIntegrateColor(True); lab.setColorMode("LAB")
    with pytest.raises(pkg.B200Error):
        lab.reset()
