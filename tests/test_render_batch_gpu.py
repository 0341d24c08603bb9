"""Reads into device memory: renderViewBatchDevice, queryDevice and getTSDFValueDevice, bit for bit.

* Batch against one pose: n = 1, 7 and 40 poses (40 spans two launches of 32) at downsample 1, 2 and 4, plain and coloured.
  Every image equals the restatement's render of the same pose and the single-pose renderView, NaNs in the same places.
* Other volumes: an RGBNormalized volume (K3) and the 2048^3 / 10 m case K4 of tests/dynamic_cases.py.
* Layout: the bytes of the caller's points outside xyz and the normal keep a sentinel pattern.
* Stream ordering: integrateBatchDevice followed by renderViewBatchDevice with no sync in between renders the fused volume.
* Device queries equal the host entry points, including the in/out valid flags.
* Errors: ESTATE before reset(), EINVAL for n < 1, a null pointer, a downsample too large and a bad layout."""

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests import dynamic_cases, general_cases
from tests.common import CAM, CFG_256, frames, query_points

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FBADBAD
POSES = [p for k in range(20) for p in (synth.orbit_pose(synth.S1, 5 * k + 2, 100),
                                        general_cases.random_poses(synth.S1, 20, 601)[k])]


def _engine(cfg, pool_log2=18, **extra):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    for k, x in {**cfg, **extra}.items():
        setattr(v._cfg, k, x)
    v._push()
    v.reset()
    return v


def batch_render(v, poses, ds, colored, stride=48, xyz_off=0, normal_off=16):
    """renderViewBatchDevice into torch buffers pre-filled with SENTINEL: (points [n, H, W, stride / 4] uint32, rgb or None)"""
    import torch
    W, H = v._cfg.image_width // ds, v._cfg.image_height // ds
    out = torch.full((len(poses), H, W, stride // 4), SENTINEL, dtype=torch.int32, device="cuda")
    rgb = torch.zeros((len(poses), H, W, 3), dtype=torch.uint8, device="cuda") if colored else None
    torch.cuda.synchronize()
    v.renderViewBatchDevice(poses, out.data_ptr(), stride, xyz_off, normal_off, None if rgb is None else rgb.data_ptr(), ds)
    v.sync()
    return out.cpu().numpy().view(np.uint32), (rgb.cpu().numpy() if colored else None)


def _f(words):
    return words.view(np.float32)


def assert_same_image(pts, rgb, want, want_rgb, *, xyz_off=0, normal_off=16, exact=False):
    """pts: [H, W, k] uint32 words of the batch; want: [H, W, 12] float32 in PointNormal layout.  exact: bit for bit (the
    engine's other entry points); else NaN-equal (the restatement's NaN payloads are not the device's)"""
    xyz, nrm = pts[..., xyz_off // 4: xyz_off // 4 + 3], pts[..., normal_off // 4: normal_off // 4 + 3]
    if exact:
        assert np.array_equal(xyz, want[..., :3].view(np.uint32)) and np.array_equal(nrm, want[..., 4:7].view(np.uint32))
    else:
        assert np.array_equal(_f(xyz), want[..., :3], equal_nan=True)
        assert np.array_equal(_f(nrm), want[..., 4:7], equal_nan=True)
    if want_rgb is not None:
        assert np.array_equal(rgb, want_rgb)


@pytest.fixture(scope="module")
def colour256():
    v = _engine(CFG_256, integrate_color=1)
    o = OracleVolume(**CFG_256, integrate_color=1)
    o.reset()
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        v.integrateCloud(cloud, None, pose); o.integrate(cloud, pose)
    v.sync()
    return v, o, {}


def _restated(o, cache, i, ds):
    if (i, ds) not in cache:
        cache[i, ds] = o.render(POSES[i], ds, colored=True)
    return cache[i, ds]


@pytest.mark.parametrize("colored", [False, True])
@pytest.mark.parametrize("ds", [1, 2, 4])
@pytest.mark.parametrize("n", [1, 7, 40])
def test_batch_equals_single_pose_and_restatement(colour256, n, ds, colored):
    v, o, cache = colour256
    pts, rgb = batch_render(v, POSES[:n], ds, colored)
    hits = 0
    for i in range(n):
        want, want_rgb = _restated(o, cache, i, ds)
        assert_same_image(pts[i], None if rgb is None else rgb[i], want, want_rgb if colored else None)
        one, one_rgb = v.renderColoredView(POSES[i], ds) if colored else (v.renderView(POSES[i], ds), None)
        assert_same_image(pts[i], None if rgb is None else rgb[i], one, one_rgb, exact=True)
        hits += int(np.isfinite(_f(pts[i][..., 2])).sum())
    assert hits > n * 1000 // (ds * ds)


@pytest.mark.parametrize("cid", ["K3", "K4"])
def test_other_volumes(cid):
    case = dynamic_cases.CASES[cid]
    v = _engine(case.config(), pool_log2=18)
    o = dynamic_cases.OracleAdapter(case)
    for pose, cloud in case.frames():
        v.integrateCloud(cloud, None, pose); o.integrate(cloud, pose)
    v.sync()
    poses = list(case.poses[-3:])
    ds = case.render_ds[0]
    pts, rgb = batch_render(v, poses, ds, True)
    for i, pose in enumerate(poses):
        want, want_rgb = o.render(pose, ds, True)
        assert_same_image(pts[i], rgb[i], want, want_rgb)
        one, one_rgb = v.renderColoredView(pose, ds)
        assert_same_image(pts[i], rgb[i], one, one_rgb, exact=True)
    assert np.isfinite(_f(pts[..., 2])).sum() > 1000


@pytest.mark.parametrize("stride,xyz_off,normal_off", [(48, 0, 16), (32, 16, 0), (24, 0, 12), (40, 28, 4)])
def test_layout_keeps_other_bytes(colour256, stride, xyz_off, normal_off):
    v, o, cache = colour256
    pts, _ = batch_render(v, POSES[:3], 2, False, stride, xyz_off, normal_off)
    mask = np.ones(stride // 4, bool)
    mask[xyz_off // 4: xyz_off // 4 + 3] = False
    mask[normal_off // 4: normal_off // 4 + 3] = False
    assert np.all(pts[..., mask] == SENTINEL)
    for i in range(3):
        assert_same_image(pts[i], None, v.renderView(POSES[i], 2), None, xyz_off=xyz_off, normal_off=normal_off, exact=True)


def test_render_is_stream_ordered_after_integrate():
    import torch
    stream = list(frames(synth.S1, 8, stride=5, color=True, noise_seed=21))
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in stream]
    poses = [p for p, _ in stream]
    torch.cuda.synchronize()
    H, W = CAM.height, CAM.width
    images = []
    for synced in (False, True):
        v = _engine(CFG_256, integrate_color=1)
        for lo in (0, 4):
            v.integrateBatchDevice([d.data_ptr() for d in dev[lo:lo + 4]], H, W, 32, poses[lo:lo + 4], rgba_off=16)
        if synced:
            v.sync()
        images.append(batch_render(v, POSES[:4], 1, True))
    (a, ca), (b, cb) = images
    assert np.array_equal(a, b) and np.array_equal(ca, cb)
    o = OracleVolume(**CFG_256, integrate_color=1)
    o.reset()
    for pose, cloud in stream:
        o.integrate(cloud, pose)
    want, want_rgb = o.render(POSES[0], 1, colored=True)
    assert_same_image(a[0], ca[0], want, want_rgb)


@pytest.mark.parametrize("what,mode", [(7, 0), (7, 1), (1, 0), (2, 0), (4, 0), (3, 1)])
def test_query_device_equals_host(colour256, what, mode):
    import torch
    v = colour256[0]
    pts = query_points(seed=3)
    n = len(pts)
    val, grad, hess, ok = v._query(pts, what, mode)
    d_xyz = torch.from_numpy(pts).cuda()
    d_val = torch.full((n,), float("nan"), device="cuda"); d_grad = torch.full((n, 3), float("nan"), device="cuda")
    d_hess = torch.full((n, 3, 3), float("nan"), device="cuda"); d_ok = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    v.queryDevice(d_xyz.data_ptr(), n, d_ok.data_ptr(), what, mode, d_val.data_ptr() if what & 1 else None,
                  d_grad.data_ptr() if what & 2 else None, d_hess.data_ptr() if what & 4 else None)
    v.sync()
    assert np.array_equal(d_ok.cpu().numpy().astype(bool), ok) and ok.sum() > 1000
    for k, (d, h) in enumerate(((d_val, val), (d_grad, grad), (d_hess, hess))):
        d = d.cpu().numpy()
        assert np.isnan(d[~ok]).all()                          # outputs of a point that is not ok are left as they were
        if what & (1 << k):
            assert np.array_equal(d[ok].view(np.uint32), h[ok].view(np.uint32))


def test_tsdf_value_device_equals_host(colour256):
    import torch
    v = colour256[0]
    pts = query_points(seed=4)
    n = len(pts)
    valid_in = (np.random.default_rng(5).random(n) < 0.8).astype(np.uint8)     # cleared flags must stay cleared
    val, ok = np.zeros(n, np.float32), valid_in.copy()
    v._check(v._lib.b200tsdf_interpolate(v._h, pts.ctypes.data, n, val.ctypes.data, ok.ctypes.data))
    d_xyz = torch.from_numpy(pts).cuda(); d_val = torch.zeros(n, device="cuda"); d_ok = torch.from_numpy(valid_in).cuda()
    torch.cuda.synchronize()
    v.getTSDFValueDevice(d_xyz.data_ptr(), n, d_val.data_ptr(), d_ok.data_ptr())
    v.sync()
    assert np.array_equal(d_ok.cpu().numpy(), ok) and 1000 < ok.sum() < valid_in.sum()
    assert np.array_equal(d_val.cpu().numpy().view(np.uint32), val.view(np.uint32))


def _code(fn):
    with pytest.raises(pkg.B200Error) as e:
        fn()
    return str(e.value).rsplit("(code ", 1)[1].rstrip(")")


def test_errors(colour256):
    import torch
    v = colour256[0]
    buf = torch.zeros(CAM.height * CAM.width * 12 * 2, dtype=torch.float32, device="cuda")
    p = buf.data_ptr()
    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    assert _code(lambda: fresh.renderViewBatchDevice(POSES[:1], p)) == "-5"
    assert _code(lambda: fresh.queryDevice(p, 4, p + 64)) == "-5"
    assert _code(lambda: fresh.getTSDFValueDevice(p, 4, p + 64, p + 128)) == "-5"
    assert _code(lambda: v.renderViewBatchDevice([], p)) == "-1"
    assert _code(lambda: v.renderViewBatchDevice(POSES[:1], 0)) == "-1"
    assert _code(lambda: v.renderViewBatchDevice(POSES[:1], p, downsampleBy=481)) == "-1"
    assert _code(lambda: v.renderViewBatchDevice(POSES[:1], p, downsampleBy=0)) == "-1"
    for stride, xo, no in ((8, 0, 0), (48, 40, 16), (48, 0, 38), (50, 0, 16), (48, 2, 16), (48, -4, 16)):
        assert _code(lambda: v.renderViewBatchDevice(POSES[:1], p, stride, xo, no)) == "-1"
    assert _code(lambda: v.renderViewBatchDevice(POSES[:1], p + 2)) == "-1"
    assert _code(lambda: v.queryDevice(0, 4, p)) == "-1"
    assert _code(lambda: v.queryDevice(p, 4, p + 64, what=1)) == "-1"              # value requested without a buffer
    assert _code(lambda: v.getTSDFValueDevice(p, 4, 0, p)) == "-1"
    v.sync()
    assert v.renderViewBatchDevice(POSES[:1], p)                                     # the handle still works
    v.sync()
