"""Tracking on the device (DESIGN.md §3i) against the host emulation of track.cuh (tests/emu/track_emu.cpp), bit for bit.

* trackDepth, trackDepthDevice and trackCloudDevice return the emulation's pose, status, iteration counts, inliers, rms, A, b
  and per-iteration log: uint16, float32 and cloud input; strides 1, 2 and 4; 640 x 480 and 643 x 479; volumes fused by the
  brick route (256^3 and 512^3, with and without colour) and by the general kernel (RGBNormalized + track_variance).
* The same call twice gives the same bytes.
* The volume is untouched: nodes, change epoch and isEmpty; and integrates interleaved with tracking calls, without a sync,
  leave the nodes of a handle that never tracked.
* Refused calls change nothing; ESTATE before reset and on a sharded handle."""
import ctypes as C
import functools

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import DEPTH_F32, DEPTH_U16, TrackParams
from tests.common import CAM, CFG_256, CFG_512
from tests.emu import track_py
from tests.test_depth_images import depth_frame
from tests.test_frame_intake_gpu import camera, device, engine, frame, ok

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL, ESTATE = -1, -5
SCHEDULES = {"default": None, "stride2": dict(levels=1, stride=[2], iters=[6]), "fine": dict(levels=2, stride=[4, 1], iters=[3, 2])}


def perturb(pose, rot_deg, trans_m):
    d = np.eye(4)
    d[:3, :3] = Rotation.from_rotvec(np.radians(rot_deg)).as_matrix()
    d[:3, 3] = trans_m
    return d @ pose


@functools.lru_cache(maxsize=None)
def volumes(case):
    """(device handle, emulated volume) fused with the same six frames"""
    cfg, color, (w, h), general = CASES[case]
    cam = camera(w, h) if (w, h) != (640, 480) else CAM
    if general:
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=18, track_variance=True)
        v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
        v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
        v.setIntegrateColor(True)
        v.setColorMode("RGBNormalized")
        v.setImageSize(cam.width, cam.height)
        v.setCameraIntrinsics(cam.fx, cam.fy, cam.cx, cam.cy)
        v.reset()
    else:
        v = engine(cfg, color, cam)
    # the emulation fuses the same {d, w} (the colour payload, which tracking does not read, is plain RGB there)
    e = track_py.TrackEmuVolume(xres=cfg["xres"], yres=cfg["yres"], zres=cfg["zres"], xsize=cfg["xsize"], ysize=cfg["ysize"],
                                zsize=cfg["zsize"], integrate_color=int(color), track_variance=int(general), fx=cam.fx, fy=cam.fy,
                                cx=cam.cx, cy=cam.cy, image_width=cam.width, image_height=cam.height, pool_log2=17)
    e.reset()
    for k in range(6):
        p, c = frame(k, cam)
        v.integrateCloud(c, None, p)
        e.integrate(c, p)
    ok(v, v._lib.b200tsdf_sync(v._h), case)
    a, b = e.dump_nodes(), v.download_nodes()
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["dw"].view(np.uint32), b["dw"].view(np.uint32)), case
    return v, e, cam


CASES = {
    "256_640": (CFG_256, False, (640, 480), False),
    "256_rgb_643": (CFG_256, True, (643, 479), False),
    "512_rgb_640": (CFG_512, True, (640, 480), False),
    "512_643": (CFG_512, False, (643, 479), False),
    "general_640": (CFG_256, True, (640, 480), True),
}


def inputs(cam, k=8):
    """ground truth, start pose and the frame in its three forms: (kind, array, scale)"""
    gt, c = frame(k, cam)
    d16, _ = depth_frame(c)
    return gt, perturb(gt, [1.0, -1.0, 0.5], [0.01, -0.01, 0.015]), [
        ("u16", d16, 1e-3), ("f32", np.ascontiguousarray(c[..., 2]), 1.0), ("cloud", np.ascontiguousarray(c), None)]


def run(v, kind, arr, scale, p0, prm):
    if kind == "cloud":
        d, = device([arr])
        return v.trackCloudDevice(d.data_ptr(), p0, prm, stride=arr.shape[2] * 4, xyz_off=0)
    if kind == "u16":
        return v.trackDepth(arr, p0, prm, depth_scale=scale)
    d, = device([arr])
    return v.trackDepthDevice(d.data_ptr(), p0, prm, depth_format=DEPTH_F32, depth_scale=scale)


def emulate(e, kind, arr, scale, p0, prm):
    if kind == "cloud":
        return e.track(arr, p0, prm)
    return e.track(arr, p0, prm, depth_scale=scale)


def same_result(a, b, what):
    (pa, ra), (pb, rb) = a, b
    assert np.array_equal(pa.view(np.uint64), pb.view(np.uint64)), (what, pa - pb)
    for k in ("status", "iters", "inliers"):
        assert ra[k] == rb[k], (what, k, ra[k], rb[k])
    assert np.float64(ra["rms"]).view(np.uint64) == np.float64(rb["rms"]).view(np.uint64), what
    assert np.array_equal(ra["A"].view(np.uint64), rb["A"].view(np.uint64)), what
    assert np.array_equal(ra["b"].view(np.uint64), rb["b"].view(np.uint64)), what
    assert ra["log"].tobytes() == rb["log"].tobytes(), what


@pytest.mark.parametrize("case", list(CASES))
def test_device_equals_emulation(case):
    v, e, cam = volumes(case)
    gt, p0, forms = inputs(cam)
    for sname, sched in SCHEDULES.items():
        prm = TrackParams.default() if sched is None else TrackParams.default(**sched)
        for kind, arr, scale in forms:
            got = run(v, kind, arr, scale, p0, prm)
            same_result(got, emulate(e, kind, arr, scale, p0, prm), f"{case} {sname} {kind}")
            assert got[1]["inliers"] > 1000 and got[1]["status"] in (pkg.TRACK_CONVERGED, pkg.TRACK_MAX_ITERS)
            same_result(run(v, kind, arr, scale, p0, prm), got, f"{case} {sname} {kind}: second call")
    # the default schedule moves towards the ground truth
    pose, res = run(v, "f32", forms[1][1], 1.0, p0, TrackParams.default())
    assert np.linalg.norm(pose[:3, 3] - gt[:3, 3]) < 0.5 * np.linalg.norm(p0[:3, 3] - gt[:3, 3]), case


def test_stop_statuses_equal_emulation():
    v, e, cam = volumes("256_640")
    gt, p0, forms = inputs(cam)
    kind, arr, scale = forms[1]
    few = TrackParams.default(min_inliers=10 ** 8)
    got = run(v, kind, arr, scale, p0, few)
    same_result(got, emulate(e, kind, arr, scale, p0, few), "too few inliers")
    assert got[1]["status"] == pkg.TRACK_TOO_FEW_INLIERS and np.array_equal(got[0], p0) and got[1]["iters"] == [1, 0, 0, 0]
    far = np.eye(4); far[:3, 3] = [0.0, 0.0, 50.0]                        # every point outside the volume: A = 0
    got = run(v, kind, arr, scale, far, TrackParams.default(min_inliers=0))
    same_result(got, emulate(e, kind, arr, scale, far, TrackParams.default(min_inliers=0)), "singular")
    assert got[1]["status"] == pkg.TRACK_SINGULAR and got[1]["inliers"] == 0
    none = TrackParams.default(iters=[0, 0, 0])
    got = run(v, kind, arr, scale, p0, none)
    assert got[1]["status"] == pkg.TRACK_MAX_ITERS and np.array_equal(got[0], p0) and len(got[1]["log"]) == 0


def test_tracking_leaves_the_volume_untouched():
    cam = CAM
    a, b = engine(CFG_256, True, cam), engine(CFG_256, True, cam)
    p0, c0 = frame(0, cam)
    for v in (a, b):
        v.integrateCloud(c0, None, p0)
        ok(v, v._lib.b200tsdf_sync(v._h))
    nodes, (epoch, _), empty = a.download_nodes(), a.changedCells(0), a.isEmpty()
    gt, start, forms = inputs(cam, 3)
    for kind, arr, scale in forms:
        run(a, kind, arr, scale, start, None)
    after = a.download_nodes()
    for k in nodes:
        assert np.array_equal(np.asarray(nodes[k]).view(np.uint8), np.asarray(after[k]).view(np.uint8)), k
    assert a.changedCells(0)[0] == epoch and a.isEmpty() == empty
    # batched depth integrates with tracking calls between them, no sync by the caller: the nodes of a handle that never tracked
    fs = [frame(k, cam) for k in range(1, 9)]
    d16 = [depth_frame(c)[0] for _, c in fs]
    dd = device(d16)
    for i in range(0, 8, 2):
        for v in (a, b):
            v.integrateDepthBatchDevice([x.data_ptr() for x in dd[i:i + 2]], [p for p, _ in fs[i:i + 2]], depth_format=DEPTH_U16,
                                        depth_scale=1e-3)
        a.trackDepthDevice(dd[i].data_ptr(), perturb(fs[i][0], [0.5, 0, 0], [0.01, 0, 0]), None, depth_format=DEPTH_U16,
                           depth_scale=1e-3)
        a.trackDepth(d16[i + 1], fs[i + 1][0])
    for v in (a, b):
        ok(v, v._lib.b200tsdf_sync(v._h))
    na, nb = a.download_nodes(), b.download_nodes()
    for k in na:
        assert np.array_equal(np.asarray(na[k]).view(np.uint8), np.asarray(nb[k]).view(np.uint8)), k
    assert a.changedCells(0)[0] == b.changedCells(0)[0] and a.stats().n_updates == b.stats().n_updates


def call(v, fn, *args):
    """fn (h, *args[:-1], params, result, no log): the raw return code"""
    prm, res = args[-1], pkg.TrackResult()
    return fn(v._h, *args[:-1], C.byref(prm) if prm is not None else None, C.byref(res), None)


def test_refusals_change_nothing():
    v, e, cam = volumes("256_640")
    gt, p0, forms = inputs(cam)
    kind, arr, scale = forms[2]
    d, = device([arr])
    want = run(v, kind, arr, scale, p0, None)
    lib = v._lib
    pose = np.ascontiguousarray(p0)
    W, H = cam.width, cam.height
    cloud = lambda *a: call(v, lib.b200tsdf_track_cloud_device, *a)
    good = dict(ptr=C.c_void_p(d.data_ptr()), stride=32, off=0, W=W, H=H, pose=pose.ctypes.data)
    bad_params = [dict(levels=0), dict(levels=5), dict(stride=[0, 2, 1]), dict(iters=[65, 1, 1]), dict(iters=[-1, 1, 1]),
                  dict(huber_delta=0.0), dict(huber_delta=float("inf")), dict(d_max=0.0), dict(d_max=float("nan")),
                  dict(w_min=float("nan")), dict(damping=-1.0), dict(eps_rot=float("inf")), dict(eps_trans=-1e-9),
                  dict(min_inliers=-1)]
    for bad in bad_params:
        assert cloud(good["ptr"], 32, 0, W, H, good["pose"], TrackParams.default(**bad)) == EINVAL, bad
    nan_pose = pose.copy(); nan_pose[0, 3] = np.nan
    assert cloud(good["ptr"], 32, 0, W, H, nan_pose.ctypes.data, TrackParams.default()) == EINVAL
    assert cloud(good["ptr"], 32, 0, W, H, None, TrackParams.default()) == EINVAL
    assert cloud(good["ptr"], 32, 0, W, H, good["pose"], None) == EINVAL
    assert cloud(None, 32, 0, W, H, good["pose"], TrackParams.default()) == EINVAL
    assert cloud(C.c_void_p(d.data_ptr() + 2), 32, 0, W, H, good["pose"], TrackParams.default()) == EINVAL
    assert cloud(good["ptr"], 30, 0, W, H, good["pose"], TrackParams.default()) == EINVAL
    assert cloud(good["ptr"], 32, 2, W, H, good["pose"], TrackParams.default()) == EINVAL
    assert cloud(good["ptr"], 32, 0, W + 1, H, good["pose"], TrackParams.default()) == EINVAL
    d16, = device([forms[0][1]])
    dep = lambda *a: call(v, lib.b200tsdf_track_depth_device, *a)
    assert dep(C.c_void_p(d16.data_ptr()), 3, C.c_float(1e-3), W, H, good["pose"], TrackParams.default()) == EINVAL
    assert dep(C.c_void_p(d16.data_ptr()), DEPTH_U16, C.c_float(0.0), W, H, good["pose"], TrackParams.default()) == EINVAL
    assert dep(C.c_void_p(d16.data_ptr() + 1), DEPTH_U16, C.c_float(1e-3), W, H, good["pose"], TrackParams.default()) == EINVAL
    assert dep(C.c_void_p(d16.data_ptr()), DEPTH_U16, C.c_float(1e-3), W, H - 1, good["pose"], TrackParams.default()) == EINVAL
    host = lambda *a: call(v, lib.b200tsdf_track_depth, *a)
    assert host(None, DEPTH_U16, C.c_float(1e-3), W, H, good["pose"], TrackParams.default()) == EINVAL
    same_result(run(v, kind, arr, scale, p0, None), want, "after refusals")
    # before reset, and on a shard
    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    assert call(fresh, lib.b200tsdf_track_depth, forms[0][1].ctypes.data, DEPTH_U16, C.c_float(1e-3), W, H, good["pose"],
                TrackParams.default()) == ESTATE
    shard = pkg.TSDFVolumeOctree(device=0, pool_log2=14, shard_rank=0, shard_count=2)
    shard.reset()
    assert call(shard, lib.b200tsdf_track_cloud_device, good["ptr"], 32, 0, W, H, good["pose"], TrackParams.default()) == ESTATE
    assert call(shard, lib.b200tsdf_track_depth_device, C.c_void_p(d16.data_ptr()), DEPTH_U16, C.c_float(1e-3), W, H, good["pose"],
                TrackParams.default()) == ESTATE
