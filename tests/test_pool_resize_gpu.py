"""Resizing a live volume's brick pool on the device (b200tsdf_resize_pool, k_pool_rehash) on a real H100.

* Every integrate route resizes mid-stream: the pool grows after frame 10, shrinks after frame 20, and the stream goes on to
  frame 30.  Frames arrive through integrate, integrateBatchDevice (two frames per call before and after each resize, so a
  graph that kept the old storage would replay it) and integrateUnorganizedBatchDevice.  After each resize and at the end
  the volume equals the oracle's nodes and, bit for bit, a handle created with the final pool: nodes, update counts,
  RGBNormalized payload, a coloured render, the mesh, both leaf lists and the .vol bytes.
* Raw storage: every claimed brick of the old pool is in the new one with its payload, the fresh invariant holds, and the
  grown pool takes new bricks as a handle created with it does.
* Shards: one shard of a pair grows and the other shrinks; their union is still the unsharded oracle's volume.
* Refusals (a pool below the load limit, one that cannot be allocated, out of range, no volume, an error latched by an
  earlier frame) change nothing: the next frame still equals the oracle.
* The C++ shim: grow, integrate and mesh."""
import os
import subprocess

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.edits_py import EditsOracleVolume
from oracle.oracle_py import OracleVolume
from tests import dynamic_cases
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, assert_same_nodes
from tests.common import frames as scene_frames
from tests.test_dynamic_scenes_gpu import EngineAdapter, check_fresh_invariant, decode_shard
from tests.test_frame_intake_gpu import Routes, camera, frame

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL, ENOMEM, ESTATE = -1, -4, -5
CAMS = camera(320, 240)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# route -> (grid, debug_flags, colour mode, track_variance, writes before the first resize)
ROUTES = {
    "fast_2048": (CFG_2048, 0, None, False, False),
    "supercell_512": (CFG_512, 0, None, False, False),
    "per_level": (CFG_512, 2, None, False, False),
    "general": (CFG_512, 1, None, False, False),
    "rgbn": (CFG_256, 0, "RGBNormalized", False, False),
    "variance": (CFG_256, 0, None, True, False),
    "written": (CFG_512, 0, None, False, True),
}
# (pool at the start, after frame 10, after frame 20): the handle it is compared with has the last one from the start
POOLS = (17, 19, 18)
# ten frames per segment: two-frame device batches, single frames and an unorganised batch
SEGMENT = ("batch_device", "cloud", "batch_device", "unorg_batch", "batch_device", "cloud")


def engine(cfg, flags, mode, var, pool):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool, track_variance=var)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
    v.setIntegrateColor(True)
    if mode:
        v.setColorMode(mode)
    v._cfg.debug_flags = flags
    v._push()
    v.setImageSize(CAMS.width, CAMS.height)
    v.setCameraIntrinsics(CAMS.fx, CAMS.fy, CAMS.cx, CAMS.cy)
    v.reset()
    return v


def oracle(cfg, mode, edits):
    kw = dict(dict(cfg, cx=CAMS.cx, cy=CAMS.cy), fx=CAMS.fx, fy=CAMS.fy, image_width=CAMS.width, image_height=CAMS.height,
              integrate_color=1, color_mode=1 if mode else 0)
    o = (EditsOracleVolume if edits else OracleVolume)(**kw)
    o.reset()
    return o


def run_segment(vols, o, k0):
    """frames k0 .. k0 + 9 through SEGMENT on every handle of vols; the oracle integrates what they were given"""
    k = k0
    for name in SEGMENT:
        routes = [Routes(v, CAMS) for v in vols]
        fs = [frame(j, CAMS) for j in range(k, k + routes[0].frames_of(name))]
        given = [r.run(name, fs) for r in routes][0]
        for pose, cloud in given:
            o.integrate(cloud, pose)
        for v in vols:
            v.sync()
        k += len(fs)
    assert k == k0 + 10


def same_everything(a, b, o, what, var, rgbn, tmp_path):
    """a against the oracle's nodes, and bit for bit against b: nodes, update counts, RGBNormalized payload, render, mesh,
    leaf lists, .vol bytes"""
    a.sync(); b.sync()
    na, nb = a.download_nodes(), b.download_nodes()
    try:
        assert_same_nodes(o.dump_nodes(), na, rgb=True, var=var)
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None
    assert na.keys() == nb.keys() and ("rgbn" in na) == bool(rgbn)   # (download_nodes carries the RGBNormalized payload)
    for k in na:
        assert np.array_equal(na[k].view(np.uint8), nb[k].view(np.uint8)), (what, k)
    assert a.stats().n_updates == b.stats().n_updates, what
    pose = frame(3, CAMS)[0]
    (ra, ca), (rb, cb) = a.renderColoredView(pose), b.renderColoredView(pose)
    assert np.array_equal(np.asarray(ra).view(np.uint8), np.asarray(rb).view(np.uint8)) and np.array_equal(ca, cb), what
    meshes = []
    for v in (a, b):
        mc = pkg.MarchingCubesTSDFOctree()
        mc.setInputTSDF(v)
        mc.setMinWeight(2.0)
        meshes.append(mc.reconstruct())
    assert len(meshes[0][0]) > 0, what
    for x, y in zip(*meshes):
        assert (x is None and y is None) or np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), what
    assert np.array_equal(a.getVoxelCenters().view(np.uint8), b.getVoxelCenters().view(np.uint8)), what
    assert np.array_equal(a.getOccupiedVoxelIndices(), b.getOccupiedVoxelIndices()), what
    pa, pb = tmp_path / "a.vol", tmp_path / "b.vol"
    a.save(str(pa)); b.save(str(pb))
    assert pa.read_bytes() == pb.read_bytes(), what


def resize(v, lg):
    v.resizePool(lg)
    st = v.stats()
    assert st.pool_capacity == 1 << lg and v._cfg.pool_log2 == lg
    print(f"  pool 2^{lg}: {st.n_bricks} bricks, load {st.n_bricks / st.pool_capacity:.3f}")


@pytest.mark.parametrize("route", list(ROUTES))
def test_resize_mid_stream(route, tmp_path):
    cfg, flags, mode, var, edits = ROUTES[route]
    a = engine(cfg, flags, mode, var, POOLS[0])
    b = engine(cfg, flags, mode, var, POOLS[-1])
    o = oracle(cfg, mode, edits)
    run_segment([a, b], o, 0)
    if edits:
        rng = np.random.default_rng(7)
        pts = rng.uniform(-1.2, 1.2, (4000, 3)).astype(np.float32)
        d, w = np.full(4000, 0.25, np.float32), np.full(4000, 3.0, np.float32)
        want = o.set_containing_voxels(pts, d, w)
        for v in (a, b):
            assert np.array_equal(v.setContainingVoxelsData(pts, d, w), want)
        assert (want == 0).sum() > 1000
    for seg, lg in enumerate(POOLS[1:], 1):
        resize(a, lg)
        same_everything(a, b, o, f"{route} after the resize to 2^{lg}", var, mode, tmp_path)
        run_segment([a, b], o, 10 * seg)
    same_everything(a, b, o, f"{route} at frame 30", var, mode, tmp_path)
    if not edits:
        assert a.stats().n_updates == o.stats().n_add_observation


def test_raw_storage_after_resize():
    """K4 (2048^3 / 10 m, colour): its coarse cells are the root arrays, so b200tsdf_export_shard lists every claimed brick
    of an unsharded handle.  The pool grows and then shrinks to the smallest that fits: the bricks and roots are the same bit
    for bit, the fresh invariant holds, and the rest of the stream claims new bricks in the moved pool as in a handle that
    never moved."""
    case = dynamic_cases.CASES["K4"]
    a, b = EngineAdapter(case, pool=15), EngineAdapter(case, pool=15)
    fr = list(case.frames())
    half = len(fr) // 2
    for pose, cloud in fr[:half]:
        a.integrate(cloud, pose); b.integrate(cloud, pose)
    before = decode_shard(a.v.export_shard().tobytes())
    n = a.v.stats().n_bricks
    small = 8
    while n * 8 > 7 << small:
        small += 1
    for lg in (17, small):
        a.v.resizePool(lg)
        after = decode_shard(a.v.export_shard().tobytes())
        assert np.array_equal(before[1], after[1])
        order_b, order_a = np.argsort(before[2]["key"]), np.argsort(after[2]["key"])
        assert np.array_equal(before[2][order_b].view(np.uint8), after[2][order_a].view(np.uint8))
        check_fresh_invariant(a.v.export_shard().tobytes())
    a.v.resizePool(small + 1)
    for pose, cloud in fr[half:]:
        a.integrate(cloud, pose); b.integrate(cloud, pose)
    na, nb = a.v.download_nodes(), b.v.download_nodes()
    for k in na:
        assert np.array_equal(na[k].view(np.uint8), nb[k].view(np.uint8)), k
    assert a.v.stats().n_bricks == b.v.stats().n_bricks > n
    print("K4 bricks at half", n, "smallest pool 2^%d" % small, "at the end", a.v.stats().n_bricks)


def test_shards_resize_on_their_own():
    from tests.shard_worker import cell_owner
    o = OracleVolume(**CFG_256); o.reset()
    shards = []
    for r in range(2):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=16, shard_rank=r, shard_count=2)
        v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy); v.reset()
        shards.append(v)
    for f, (pose, cloud) in enumerate(scene_frames(synth.S1, 4, stride=11, noise_seed=21)):
        o.integrate(cloud, pose)
        for v in shards:
            v.integrateCloud(cloud, None, pose)
        if f == 1:
            shards[0].resizePool(18)
            shards[1].resizePool(15)
    ref = o.dump_nodes()
    C = o.levels()[0]
    owner = np.array([cell_owner(*c, 2) for c in (ref["keys"][:, 1:] >> (ref["keys"][:, 0:1] - C))])
    for r, v in enumerate(shards):
        d = v.download_nodes()
        own = np.array([cell_owner(*c, 2) for c in (d["keys"][:, 1:] >> (d["keys"][:, 0:1] - C))]) == r
        assert np.array_equal(d["keys"][own], ref["keys"][owner == r])
        assert np.array_equal(d["dw"][own].view(np.uint32), ref["dw"][owner == r].view(np.uint32))
    assert [v.stats().pool_capacity for v in shards] == [1 << 18, 1 << 15]


def _raises(code, call):
    with pytest.raises(pkg.B200Error, match=rf"\(code {code}\)"):
        call()


def test_refusals_change_nothing():
    v = engine(CFG_512, 0, None, False, 17)
    o = oracle(CFG_512, None, False)
    fs = [frame(k, CAMS) for k in range(4)]
    for pose, cloud in fs[:3]:
        v.integrateCloud(cloud, None, pose); o.integrate(cloud, pose)
    n = v.stats().n_bricks
    assert n > 224
    nodes = v.download_nodes()

    def unchanged():
        after = v.download_nodes()
        for k in nodes:
            assert np.array_equal(nodes[k].view(np.uint8), after[k].view(np.uint8)), k
        st = v.stats()
        assert st.pool_capacity == 1 << 17 and st.n_bricks == n and v._cfg.pool_log2 == 17

    _raises(EINVAL, lambda: v.resizePool(8))            # below the load limit
    unchanged()
    _raises(ENOMEM, lambda: v.resizePool(26))           # about 313 GB: the allocation is refused
    unchanged()
    _raises(EINVAL, lambda: v.resizePool(27))
    unchanged()
    pose, cloud = fs[3]
    v.integrateCloud(cloud, None, pose); o.integrate(cloud, pose)
    v.sync()
    assert_same_nodes(o.dump_nodes(), v.download_nodes(), rgb=True)
    assert v.stats().n_updates == o.stats().n_add_observation

    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    _raises(ESTATE, lambda: fresh.resizePool(16))       # no volume yet

    small = pkg.TSDFVolumeOctree(device=0, pool_log2=8)  # overflows in its first frame: the volume is incomplete
    small.setResolution(512, 512, 512); small.setCameraIntrinsics(525, 525, CAM.cx, CAM.cy); small.reset()
    pose = synth.orbit_pose(synth.S1, 0, 1)
    with pytest.raises(pkg.B200Error):
        small.integrateCloud(synth.make_frame(synth.S1, pose, CAM), None, pose)
        small.sync()
    _raises(ESTATE, lambda: small.resizePool(18))


def test_cpp_shim_resize(engine_lib, tmp_path):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(tmp_path), "shim_resize")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-O1", os.path.join(ROOT, "tests", "cpp", "shim_resize.cpp"), "-o", exe, f"-L{libdir}",
                    "-lb200tsdf", f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "mesh:" in r.stdout
