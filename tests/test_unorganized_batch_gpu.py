"""b200tsdf_integrate_unorganized_batch_device: n unorganised clouds resident in device memory, organised and fused 32 per graph
launch, must equal n calls of b200tsdf_integrate_unorganized on the same clouds and the oracle (the restatement's organise of
each cloud followed by its integrate) in every node, colour, M / ns and RGBNormalized payload."""
import ctypes as C

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle import oracle_py
from tests.common import CAM, CFG_256, CFG_2048, assert_same_nodes, frames
from tests.test_organize import INTR, unorganized_cloud

pytestmark = pytest.mark.gpu

EINVAL, ESTATE = -1, -5
_BASE = {}


def _base(seed, color, scale=1.0, world=None):
    key = (seed, color, scale, None if world is None else world.tobytes())
    if key not in _BASE:
        _BASE[key] = unorganized_cloud(seed, color=color, scale=scale, world_pose=world)[0]
    return _BASE[key]


def make_clouds(n, *, color=True, empty=(), seed0=0, scale=1.0, worlds=None):
    """n shuffled unorganised clouds with different points and counts; the frames listed in `empty` have no points"""
    out = []
    for i in range(n):
        k = seed0 + i
        b = _base(30 + k % 4, color, scale, None if worlds is None else worlds[i])
        if i in empty:
            out.append(np.zeros((0, b.shape[1]), np.float32))
            continue
        rng = np.random.default_rng(100 + k)
        out.append(np.ascontiguousarray(b[rng.permutation(len(b))[: len(b) - 1499 * (k % 17)]]))
    return out


def poses_for(n, seed0=0):
    return [synth.orbit_pose(synth.S1, 3 + 2 * ((seed0 + i) % 40), 100) for i in range(n)]


def engine(cfg, pool_log2=17, *, color=False, track_variance=False, color_mode=0):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, track_variance=track_variance)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
    v.setCameraIntrinsics(525.0, 525.0, cfg["cx"], cfg["cy"])
    v.setIntegrateColor(color)
    v._cfg.color_mode = color_mode; v._push()
    v.reset()
    return v


def oracle(cfg, *, color=False, color_mode=0):
    o = oracle_py.OracleVolume(**cfg, integrate_color=int(color), color_mode=color_mode)
    o.reset()
    return o


def opts(units=1.0, zero_nans=False, w2c=None):
    tf = None if w2c is None else np.ascontiguousarray(w2c, np.float64)
    return pkg.OrganizeOpts(float(units), int(zero_nans), None if tf is None else tf.ctypes.data), tf


def host_calls(v, clouds, poses, rgba_off, units=1.0, zero_nans=False, w2cs=None):
    """one b200tsdf_integrate_unorganized per cloud (host points)"""
    for i, c in enumerate(clouds):
        o, _keep = opts(units, zero_nans, None if w2cs is None else w2cs[i])
        pose = np.ascontiguousarray(poses[i], np.float64)
        rc = v._lib.b200tsdf_integrate_unorganized(v._h, c.ctypes.data if len(c) else None, len(c), c.shape[1] * 4, 0, rgba_off,
                                                   C.byref(o), pose.ctypes.data)
        assert rc == 0, v._lib.b200tsdf_last_error(v._h)


def upload(clouds):
    import torch
    dev = [torch.from_numpy(c).cuda() if len(c) else None for c in clouds]
    torch.cuda.synchronize()
    return dev, [0 if d is None else d.data_ptr() for d in dev]


def device_batch(v, clouds, poses, rgba_off, units=1.0, zero_nans=False, w2cs=None, sync=True):
    dev, ptrs = upload(clouds)
    v.integrateUnorganizedBatchDevice(ptrs, [len(c) for c in clouds], clouds[0].shape[1] * 4, poses, rgba_off=rgba_off,
                                      cloud_units=units, zero_nans=zero_nans, worlds_to_camera=w2cs)
    if sync:
        v.sync()
    return dev                                                    # (the caller keeps the clouds alive until a sync)


def oracle_calls(o, clouds, poses, rgba_off, units=1.0, zero_nans=False, w2cs=None):
    for i, c in enumerate(clouds):
        org, _ = oracle_py.organize(c, INTR, CAM.width, CAM.height, rgba_off=rgba_off, cloud_units=units, zero_nans=zero_nans,
                                    world_to_camera=None if w2cs is None else w2cs[i])
        o.integrate(org, poses[i])


# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 32, 45])
def test_batch_equals_host_calls_and_oracle(n):
    clouds = make_clouds(n, empty=() if n == 1 else (n // 2,))
    poses = poses_for(n)
    v, ref, o = engine(CFG_256, color=True), engine(CFG_256, color=True), oracle(CFG_256, color=True)
    device_batch(v, clouds, poses, 16)
    host_calls(ref, clouds, poses, 16)
    oracle_calls(o, clouds, poses, 16)
    if n == 45:
        # a second call replays the graphs captured by the first (both record halves)
        more = make_clouds(n, seed0=7, empty=(3,)); mp = poses_for(n, seed0=5)
        device_batch(v, more, mp, 16); host_calls(ref, more, mp, 16); oracle_calls(o, more, mp, 16)
    a = v.download_nodes()
    assert_same_nodes(ref.download_nodes(), a, rgb=True)
    assert_same_nodes(o.dump_nodes(), a, rgb=True)


@pytest.mark.parametrize("color,point_floats,rgba_off", [(True, 8, -1), (False, 4, -1), (True, 4, 12), (False, 8, 16)])
def test_point_layouts(color, point_floats, rgba_off):
    clouds = make_clouds(5, color=point_floats == 8, empty=(1,))
    if point_floats == 4 and rgba_off >= 0:                       # 16-byte points with colour bytes in the fourth word
        rng = np.random.default_rng(3)
        for c in clouds:
            c[:, 3] = rng.integers(0, 256, (len(c), 4), dtype=np.uint8).view(np.float32)[:, 0]
    poses = poses_for(5, seed0=11)
    v, ref, o = engine(CFG_256, color=color), engine(CFG_256, color=color), oracle(CFG_256, color=color)
    device_batch(v, clouds, poses, rgba_off)
    host_calls(ref, clouds, poses, rgba_off)
    oracle_calls(o, clouds, poses, rgba_off)
    a = v.download_nodes()
    assert_same_nodes(ref.download_nodes(), a, rgb=color)
    assert_same_nodes(o.dump_nodes(), a, rgb=color)


def test_units_zero_nans_and_a_world_transform_per_frame():
    n = 6
    worlds = [synth.orbit_pose(synth.S1, 17 + 9 * i, 100) for i in range(n)]
    clouds = make_clouds(n, scale=0.001, worlds=worlds, empty=(4,))
    w2cs = [np.linalg.inv(w) for w in worlds]
    poses = poses_for(n, seed0=2)
    kw = dict(units=0.001, zero_nans=True, w2cs=w2cs)
    v, ref, o = engine(CFG_256, color=True), engine(CFG_256, color=True), oracle(CFG_256, color=True)
    device_batch(v, clouds, poses, 16, **kw)
    host_calls(ref, clouds, poses, 16, **kw)
    oracle_calls(o, clouds, poses, 16, **kw)
    a = v.download_nodes()
    assert len(a["keys"]) > 1000
    assert_same_nodes(ref.download_nodes(), a, rgb=True)
    assert_same_nodes(o.dump_nodes(), a, rgb=True)


@pytest.mark.parametrize("route", ["brick_2048", "variance_256", "rgbnorm_256"])
def test_routes_against_the_oracle(route):
    cfg, pool, kw = {"brick_2048": (CFG_2048, 18, {}), "variance_256": (CFG_256, 17, dict(track_variance=True)),
                     "rgbnorm_256": (CFG_256, 17, dict(track_variance=True, color_mode=1))}[route]
    n = 7
    clouds = make_clouds(n, empty=(2,), seed0=3)
    poses = poses_for(n, seed0=9)
    v = engine(cfg, pool, color=True, **kw)
    o = oracle(cfg, color=True, color_mode=kw.get("color_mode", 0))
    device_batch(v, clouds, poses, 16)
    oracle_calls(o, clouds, poses, 16)
    da, db = o.dump_nodes(), v.download_nodes()
    assert_same_nodes(da, db, rgb=True, var=kw.get("track_variance", False))
    if kw.get("color_mode"):
        # the RGBNormalized payload: bit for bit against one b200tsdf_integrate_unorganized per cloud, NaNs included
        ref = engine(cfg, pool, color=True, **kw)
        host_calls(ref, clouds, poses, 16)
        assert np.array_equal(ref.download_nodes()["rgbn"].view(np.uint32), db["rgbn"].view(np.uint32))
        # against the oracle: the same NaN positions and bit-identical values elsewhere (the junk points of these clouds are
        # black, whose normalised colour is NaN)
        a, b = da["rgbn"], db["rgbn"]
        nan = np.isnan(a)
        assert np.array_equal(nan, np.isnan(b)), "NaN positions of the payload differ"
        assert np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32)), "payload values differ"
        nan_bits = int((a[nan].view(np.uint32) != b[nan].view(np.uint32)).sum())
        print(f"rgbn: {int(nan.sum())} NaN floats, {nan_bits} with other bits than the oracle's")


def test_launch_accounting():
    v = engine(CFG_256, color=True)
    organised = [c for _, c in frames(synth.S1, 1, color=True)]
    dev, ptrs = upload(organised)
    v.profile_begin()
    v.integrateBatchDevice(ptrs, CAM.height, CAM.width, 32, poses_for(1), rgba_off=16)
    per_frame = v.profile_end().total_launches
    assert per_frame >= 2
    got = {}
    for n, trim in ((45, 0), (45, 200000), (32, 0)):
        clouds = [c[: len(c) - trim] for c in make_clouds(n)]
        v.profile_begin()
        keep = device_batch(v, clouds, poses_for(n), 16)
        pr = v.profile_end()
        del keep
        batches = -(-n // 32)
        assert pr.graph_launches == batches
        assert pr.total_launches == 3 * batches + n * per_frame
        assert pr.n_frames == n
        got[(n, trim)] = pr.h2d_bytes
    assert got[(45, 0)] == got[(45, 200000)] and got[(45, 0)] < 4096          # the points never cross PCIe


def test_render_right_after_a_batch_is_ordered_behind_it():
    import torch
    v = engine(CFG_256, color=True)
    clouds = make_clouds(40, empty=(6,))
    poses = poses_for(40)
    views = poses_for(4, seed0=20)
    W, H = CAM.width, CAM.height
    a = torch.zeros((4, H, W, 12), dtype=torch.float32, device="cuda")
    b = torch.zeros_like(a)
    torch.cuda.synchronize()
    keep = device_batch(v, clouds, poses, 16, sync=False)
    v.renderViewBatchDevice(views, a.data_ptr())                  # no sync in between
    v.sync()
    v.renderViewBatchDevice(views, b.data_ptr())
    v.sync()
    del keep
    x, y = a.cpu().numpy(), b.cpu().numpy()
    assert np.isfinite(y[..., 2]).sum() > 50000
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


def test_unorganised_and_organised_batches_interleave():
    v, o = engine(CFG_256, color=True), oracle(CFG_256, color=True)
    organised = list(frames(synth.S1, 6, stride=7, color=True, noise_seed=5))
    keep = []
    for step in range(2):
        part = organised[3 * step: 3 * step + 3]
        dev, ptrs = upload([c for _, c in part])
        keep.append(dev)
        clouds = make_clouds(4, seed0=5 * step, empty=(1,) if step else ())
        poses = poses_for(4, seed0=13 * step)
        if step == 0:                                            # organised, then unorganised
            v.integrateBatchDevice(ptrs, CAM.height, CAM.width, 32, [p for p, _ in part], rgba_off=16)
            keep.append(device_batch(v, clouds, poses, 16, sync=False))
            for p, c in part:
                o.integrate(c, p)
            oracle_calls(o, clouds, poses, 16)
        else:                                                    # unorganised, then organised
            keep.append(device_batch(v, clouds, poses, 16, sync=False))
            v.integrateBatchDevice(ptrs, CAM.height, CAM.width, 32, [p for p, _ in part], rgba_off=16)
            oracle_calls(o, clouds, poses, 16)
            for p, c in part:
                o.integrate(c, p)
    v.sync()
    assert_same_nodes(o.dump_nodes(), v.download_nodes(), rgb=True)


def test_refusals_leave_the_handle_usable():
    import torch
    lib = pkg.load_library()
    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    clouds = make_clouds(3)
    dev, ptrs = upload(clouds)
    poses = np.ascontiguousarray(np.stack(poses_for(3)), np.float64)
    o, _ = opts()

    def call(vol, n=3, p=ptrs, counts=None, stride=32, xyz_off=0, rgba_off=16, op=C.byref(o), ps=poses.ctypes.data):
        arr = None if p is None else (C.c_void_p * max(len(p), 1))(*[x or None for x in p])
        cnt = None if counts is False else (C.c_size_t * 3)(*(counts or [len(c) for c in clouds]))
        return lib.b200tsdf_integrate_unorganized_batch_device(vol._h, n, arr, cnt, stride, xyz_off, rgba_off, op, ps)

    assert call(fresh) == ESTATE                                   # before reset()
    v = engine(CFG_256, color=True)
    assert call(v, n=-1) == EINVAL
    assert call(v, p=None) == EINVAL
    assert call(v, counts=False) == EINVAL
    assert call(v, ps=None) == EINVAL
    assert call(v, op=None) == EINVAL
    assert call(v, p=[ptrs[0], 0, ptrs[2]]) == EINVAL               # null cloud with points
    assert call(v, counts=[len(clouds[0]), 1 << 32, 5]) == EINVAL   # 2^32 points
    for stride, xyz_off, rgba_off in ((13, 0, -1), (32, 2, 16), (32, 0, 14), (16, 8, -1), (16, 0, 16), (36, 0, 34)):
        assert call(v, stride=stride, xyz_off=xyz_off, rgba_off=rgba_off) == EINVAL, (stride, xyz_off, rgba_off)
    assert call(v, n=0) == 0
    # the same alignment rule for the host entry points, which share the kernels
    pts = np.zeros((10, 8), np.float32)
    out = np.zeros((CAM.height, CAM.width, 8), np.float32)
    assert lib.b200tsdf_organize(v._h, pts.ctypes.data, 3, 13, 0, -1, C.byref(o), out.ctypes.data, 32, 16, None) == EINVAL
    pose = np.eye(4)
    assert lib.b200tsdf_integrate_unorganized(v._h, pts.ctypes.data, 3, 13, 0, -1, C.byref(o), pose.ctypes.data) == EINVAL
    assert lib.b200tsdf_integrate_unorganized(v._h, pts.ctypes.data, 3, 32, 0, 6, C.byref(o), pose.ctypes.data) == EINVAL
    # a cloud without points may be NULL
    assert call(v, p=[ptrs[0], 0, ptrs[2]], counts=[len(clouds[0]), 0, len(clouds[2])]) == 0
    # nothing of the refused calls was enqueued: the volume equals the accepted batch alone
    v.sync()
    ref = engine(CFG_256, color=True)
    host_calls(ref, [clouds[0], clouds[1][:0], clouds[2]], list(poses), 16)
    assert_same_nodes(ref.download_nodes(), v.download_nodes(), rgb=True)
    del dev
    torch.cuda.synchronize()
