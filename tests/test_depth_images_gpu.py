"""Depth images on the engine (DESIGN.md §3h), against the oracle fed cpu_tsdf_b200.depth_to_cloud, bit for bit.

* depthToCloudDevice writes depth_to_cloud's bytes for every map of tests/test_depth_images.py.
* integrateDepth and integrateDepthBatchDevice equal the oracle on every node: uint16 and float32, with and without colour,
  256^3 / 3 m and 512^3 / 3 m with colour, 640 x 480 and 643 x 479, an RGBNormalized + track_variance volume (the general
  kernel), and batches that cross a record half (33 and 65 frames).
* Every ordered pair of the eleven routes (the nine of test_frame_intake_gpu plus the two depth routes) on one handle without
  a sync.
* Refused calls in the middle of a stream change nothing.
* The host buffers of integrateDepth are overwritten right after each call returns.
* After depth frames, IncrementalMesh.update() equals reconstructDevice, and render, mesh and .vol bytes equal those of a handle
  fed the same frames as depth_to_cloud clouds through integrateCloud."""
import ctypes as C

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import DEPTH_F32, DEPTH_U16, depth_to_cloud
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256, CFG_512, assert_same_nodes
from tests.emu.depth_py import cloud_pixels
from tests.test_depth_images import CASES, depth_frame
from tests.test_dynamic_scenes_gpu import debug_timing
from tests.test_frame_intake_gpu import Routes, camera, de_bruijn, device, engine, frame, ok, oracle, poses_arg

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL, ESTATE = -1, -5


def intr(cam):
    return (cam.fx, cam.fy, cam.cx, cam.cy)


def depth_of(cloud, fmt):
    """(depth map, scale, rgb) of a synthetic colour frame: uint16 millimetres, or float32 metres (NaN stays NaN)"""
    d16, rgb = depth_frame(cloud)
    if fmt == DEPTH_U16:
        return d16, 1e-3, rgb
    return np.ascontiguousarray(cloud[..., 2]), 1.0, rgb


def oracle_cloud(d, scale, rgb, cam, color=True):
    return depth_to_cloud(d, intr(cam), rgb if color else None, scale)


def check(v, o, what, *, rgbn=False):
    ok(v, v._lib.b200tsdf_sync(v._h), what)
    assert v.stats().n_updates == o.stats().n_add_observation, what
    a, b = o.dump_nodes(), v.download_nodes()
    assert_same_nodes(a, b, rgb=bool(v._cfg.integrate_color))
    if rgbn:
        assert np.array_equal(a["rgbn"].view(np.uint32), b["rgbn"].view(np.uint32)), what


# ---- depthToCloudDevice ------------------------------------------------------------------------------------------------
def test_depth_to_cloud_device_bytes():
    vols = {}
    for name, d, K, rgb, scale in CASES:
        H, W = d.shape
        if (W, H, K) not in vols:
            v = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
            v.setResolution(256, 256, 256)
            v.setImageSize(W, H)
            v.setCameraIntrinsics(*K)
            v.reset()
            vols[(W, H, K)] = v
        v = vols[(W, H, K)]
        dd, = device([d])
        dr = device([rgb])[0] if rgb is not None else None
        out = torch.full((H * W * 16,), 0xA5, dtype=torch.uint8, device="cuda:0")
        torch.cuda.synchronize()
        v.depthToCloudDevice(dd.data_ptr(), out.data_ptr(), depth_format=DEPTH_U16 if d.dtype == np.uint16 else DEPTH_F32,
                             depth_scale=scale, d_rgb=None if dr is None else dr.data_ptr())
        got = out.cpu().numpy().view(np.uint32).reshape(H, W, 4)
        want = cloud_pixels(depth_to_cloud(d, K, rgb, scale))
        assert np.array_equal(got, want), (name, np.argwhere(np.any(got != want, axis=-1))[:5])


# ---- parity --------------------------------------------------------------------------------------------------------------
PARITY = {
    "256_u16_640": (CFG_256, False, DEPTH_U16, (640, 480), False),
    "256_f32_643": (CFG_256, False, DEPTH_F32, (643, 479), False),
    "256_u16_rgb_ignored": (CFG_256, False, DEPTH_U16, (640, 480), True),
    "512_u16_rgb_640": (CFG_512, True, DEPTH_U16, (640, 480), True),
    "512_f32_rgb_643": (CFG_512, True, DEPTH_F32, (643, 479), True),
    "512_u16_no_rgb_643": (CFG_512, True, DEPTH_U16, (643, 479), False),
}


@pytest.mark.parametrize("case", list(PARITY))
def test_integrate_depth_and_batches_equal_the_oracle(case):
    cfg, color, fmt, (w, h), with_rgb = PARITY[case]
    cam = camera(w, h) if (w, h) != (640, 480) else CAM
    v, o = engine(cfg, color, cam), oracle(cfg, color, cam)
    k = 0
    for _ in range(5):                                       # integrateDepth, frame by frame
        p, c = frame(k, cam)
        d, scale, rgb = depth_of(c, fmt)
        v.integrateDepth(d, p, rgb if with_rgb else None, scale)
        o.integrate(oracle_cloud(d, scale, rgb, cam, with_rgb), p)
        k += 1
    check(v, o, f"{case}: integrateDepth")
    for n in (1, 4):                                         # integrateDepthBatchDevice
        fs = [frame(j, cam) for j in range(k, k + n)]
        ds = [depth_of(c, fmt) for _, c in fs]
        dd = device([d for d, _, _ in ds])
        dr = device([r for _, _, r in ds]) if with_rgb else None
        v.integrateDepthBatchDevice([x.data_ptr() for x in dd], [p for p, _ in fs], depth_format=fmt, depth_scale=ds[0][1],
                                    d_rgb_ptrs=None if dr is None else [x.data_ptr() for x in dr])
        for (p, _), (d, scale, rgb) in zip(fs, ds):
            o.integrate(oracle_cloud(d, scale, rgb, cam, with_rgb), p)
        k += n
        check(v, o, f"{case}: batch of {n}")


def test_general_kernel_rgbnormalized_track_variance():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=18, track_variance=True)
    for key, x in CFG_256.items():
        setattr(v._cfg, key, x)
    v._cfg.integrate_color, v._cfg.color_mode = 1, 1
    v._push()
    v.setImageSize(CAM.width, CAM.height)
    v.setCameraIntrinsics(*intr(CAM))
    v.reset()
    o = OracleVolume(**dict(CFG_256, cx=CAM.cx, cy=CAM.cy), fx=CAM.fx, fy=CAM.fy, image_width=CAM.width, image_height=CAM.height,
                     integrate_color=1, color_mode=1)
    o.reset()
    for k in range(4):
        p, c = frame(k)
        d, scale, rgb = depth_of(c, DEPTH_U16)
        if k < 2:
            v.integrateDepth(d, p, rgb, scale)
        else:
            dd, dr = device([d, rgb])
            v.integrateDepthBatchDevice([dd.data_ptr()], [p], depth_format=DEPTH_U16, depth_scale=scale, d_rgb_ptrs=[dr.data_ptr()])
            ok(v, v._lib.b200tsdf_sync(v._h))
        o.integrate(oracle_cloud(d, scale, rgb, CAM), p)
    check(v, o, "RGBNormalized + track_variance", rgbn=True)


@pytest.mark.parametrize("n", [33, 65])
def test_batches_across_record_halves(n):
    v, o = engine(CFG_256, True), oracle(CFG_256, True)
    fs = [frame(k % 45) for k in range(n)]
    ds = [depth_of(c, DEPTH_U16) for _, c in fs]
    dd = device([d for d, _, _ in ds])
    dr = device([r for _, _, r in ds])
    v.integrateDepthBatchDevice([x.data_ptr() for x in dd], [p for p, _ in fs], depth_format=DEPTH_U16, depth_scale=1e-3,
                                d_rgb_ptrs=[x.data_ptr() for x in dr])
    for (p, _), (d, scale, rgb) in zip(fs, ds):
        o.integrate(oracle_cloud(d, scale, rgb, CAM), p)
    check(v, o, f"batch of {n}")


# ---- switches between routes ---------------------------------------------------------------------------------------------
class DepthRoutes(Routes):
    """the nine routes plus integrateDepth (one frame, uint16 + colour from host memory) and integrateDepthBatchDevice (two
    frames, float32 + colour in device memory)"""

    ONE = Routes.ONE + ("depth_host",)
    TWO = Routes.TWO + ("depth_batch",)
    NAMES = Routes.NAMES + ("depth_host", "depth_batch")

    def depth_host(self, fs):
        (p, c), = fs
        d, scale, rgb = depth_of(c, DEPTH_U16)
        self.v.integrateDepth(d, p, rgb, scale)
        return [(p, oracle_cloud(d, scale, rgb, self.cam))]

    def depth_batch(self, fs):
        ds = [depth_of(c, DEPTH_F32) for _, c in fs]
        dd = device([d for d, _, _ in ds])
        dr = device([r for _, _, r in ds])
        self.keep.append((dd, dr))
        self.v.integrateDepthBatchDevice([x.data_ptr() for x in dd], [p for p, _ in fs], depth_format=DEPTH_F32, depth_scale=1.0,
                                         d_rgb_ptrs=[x.data_ptr() for x in dr])
        return [(p, oracle_cloud(d, scale, rgb, self.cam)) for (p, _), (d, scale, rgb) in zip(fs, ds)]


def test_every_switch_between_eleven_routes():
    walk = [DepthRoutes.NAMES[i] for i in de_bruijn(len(DepthRoutes.NAMES))]
    walk.append(walk[0])
    assert len(walk) == 122 and len(set(zip(walk, walk[1:]))) == 121
    v, o = engine(CFG_512, True), oracle(CFG_512, True)
    r = DepthRoutes(v)
    debug_timing(v)
    gated = plain = k = 0
    checkpoints = {30, 61, 92, len(walk)}
    for i, name in enumerate(walk, 1):
        fs = [frame(j % 45) for j in range(k, k + r.frames_of(name))]
        k += len(fs)
        for p, c in r.run(name, fs):
            o.integrate(c, p)
        if i in checkpoints:
            ok(v, v._lib.b200tsdf_sync(v._h))
            assert v.stats().n_updates == o.stats().n_add_observation, (i, name)
            assert_same_nodes(o.dump_nodes(), v.download_nodes(), rgb=True)
            r.keep.clear()
            dt = debug_timing(v)
            gated += int(dt[11]); plain += int(dt[12])
    assert (gated, plain) == (k - 1, 1), k


# ---- refused calls ---------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing():
    v, o = engine(CFG_512, True), oracle(CFG_512, True)
    lib, h = v._lib, v._h
    W, H = CAM.width, CAM.height
    for k in range(2):
        p, c = frame(k)
        d, scale, rgb = depth_of(c, DEPTH_U16)
        v.integrateDepth(d, p, rgb, scale)
        o.integrate(oracle_cloud(d, scale, rgb, CAM), p)
    check(v, o, "before")
    epoch0, _ = v.changedCells(0)
    nodes0 = v.download_nodes()

    p, c = frame(10)
    d16, _, rgb = depth_of(c, DEPTH_U16)
    raw = np.zeros(d16.nbytes + 8, np.uint8)
    mis = raw[1:1 + d16.nbytes]                             # a uint16 map one byte off its alignment
    mis[:] = d16.view(np.uint8).reshape(-1)
    dd, dr = device([d16, rgb])
    dbytes = torch.zeros(d16.nbytes + 16, dtype=torch.uint8, device="cuda:0")
    torch.cuda.synchronize()
    dp, rp = dd.data_ptr(), dr.data_ptr()
    ps = poses_arg([p] * 40)
    out = torch.empty(W * H * 16, dtype=torch.uint8, device="cuda:0")
    arr = lambda xs: (C.c_void_p * len(xs))(*xs)

    def host(fmt=DEPTH_U16, scale=1e-3, w=W, hh=H, ptr=None):
        return lib.b200tsdf_integrate_depth(h, C.c_void_p(d16.ctypes.data) if ptr is None else ptr, fmt, scale, rgb.ctypes.data, w, hh,
                                            ps.ctypes.data)

    def batch(n=2, ptrs=None, rgbs="same", fmt=DEPTH_U16, scale=1e-3, w=W, hh=H):
        ptrs = [dp] * n if ptrs is None else ptrs
        rg = arr([rp] * n) if rgbs == "same" else (None if rgbs is None else arr(rgbs))
        return lib.b200tsdf_integrate_depth_batch_device(h, n, arr(ptrs), fmt, scale, rg, w, hh, ps.ctypes.data)

    def cloud(fmt=DEPTH_U16, scale=1e-3, w=W, hh=H, ptr=None, o_ptr=None):
        return lib.b200tsdf_depth_to_cloud_device(h, C.c_void_p(dp) if ptr is None else ptr, fmt, scale, None, w, hh,
                                                  C.c_void_p(out.data_ptr()) if o_ptr is None else o_ptr)

    refusals = []
    for fn in (host, batch, cloud):
        nm = fn.__name__
        refusals += [
            (f"{nm} format 0", lambda fn=fn: fn(fmt=0)),
            (f"{nm} format 3", lambda fn=fn: fn(fmt=3)),
            (f"{nm} scale 0", lambda fn=fn: fn(scale=0.0)),
            (f"{nm} scale -1", lambda fn=fn: fn(scale=-1.0)),
            (f"{nm} scale nan", lambda fn=fn: fn(scale=float("nan"))),
            (f"{nm} scale inf", lambda fn=fn: fn(scale=float("inf"))),
            (f"{nm} width", lambda fn=fn: fn(w=W - 1)),
            (f"{nm} height", lambda fn=fn: fn(hh=H + 1)),
        ]
    refusals += [
        ("host null depth", lambda: lib.b200tsdf_integrate_depth(h, None, DEPTH_U16, 1e-3, None, W, H, ps.ctypes.data)),
        ("host misaligned u16", lambda: host(ptr=C.c_void_p(mis.ctypes.data))),
        ("host misaligned f32", lambda: host(fmt=DEPTH_F32, ptr=C.c_void_p(d16.ctypes.data + 2))),
        ("batch null at 1", lambda: batch(ptrs=[dp, None])),
        ("batch n=40 null at 35", lambda: batch(n=40, ptrs=[dp] * 35 + [None] + [dp] * 4)),
        ("batch null rgb entry", lambda: batch(rgbs=[rp, None])),
        ("batch n=40 null rgb at 39", lambda: batch(n=40, rgbs=[rp] * 39 + [None])),
        ("batch misaligned u16", lambda: batch(ptrs=[dp, dbytes.data_ptr() + 1])),
        ("batch misaligned f32", lambda: batch(fmt=DEPTH_F32, ptrs=[dbytes.data_ptr() + 2, dp])),
        ("cloud null depth", lambda: cloud(ptr=C.c_void_p(0))),
        ("cloud misaligned", lambda: cloud(ptr=C.c_void_p(dbytes.data_ptr() + 1))),
        ("cloud misaligned out", lambda: cloud(o_ptr=C.c_void_p(out.data_ptr() + 4))),
    ]
    for what, call in refusals:
        assert call() == EINVAL, what
        epoch, _ = v.changedCells(0)
        assert epoch == epoch0, what
    ok(v, lib.b200tsdf_sync(h))
    assert_same_nodes(nodes0, v.download_nodes(), rgb=True)
    # the stream goes on in step: the next frame of each route equals the oracle
    v.integrateDepth(d16, p, rgb, 1e-3)
    o.integrate(oracle_cloud(d16, 1e-3, rgb, CAM), p)
    ok(v, batch(n=1))
    o.integrate(oracle_cloud(d16, 1e-3, rgb, CAM), p)
    check(v, o, "after the refusals")
    assert v.changedCells(0)[0] == epoch0 + 2

    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)   # before reset ()
    assert fresh._lib.b200tsdf_integrate_depth(fresh._h, d16.ctypes.data, DEPTH_U16, 1e-3, None, W, H, ps.ctypes.data) == ESTATE
    shard = pkg.TSDFVolumeOctree(device=0, pool_log2=14, shard_rank=0, shard_count=2)
    shard.setResolution(256, 256, 256)
    shard.reset()
    sh = shard._h
    assert shard._lib.b200tsdf_integrate_depth(sh, d16.ctypes.data, DEPTH_U16, 1e-3, None, W, H, ps.ctypes.data) == ESTATE
    assert shard._lib.b200tsdf_integrate_depth_batch_device(sh, 1, arr([dp]), DEPTH_U16, 1e-3, None, W, H, ps.ctypes.data) == ESTATE
    assert shard._lib.b200tsdf_depth_to_cloud_device(sh, dp, DEPTH_U16, 1e-3, None, W, H, out.data_ptr()) == ESTATE


# ---- caller buffers ------------------------------------------------------------------------------------------------------
def test_host_buffers_overwritten_after_each_call():
    v, o = engine(CFG_512, True), oracle(CFG_512, True)
    dbuf = np.empty((CAM.height, CAM.width), np.uint16)
    cbuf = np.empty((CAM.height, CAM.width, 3), np.uint8)
    for k in range(12):
        p, c = frame(k)
        d, scale, rgb = depth_of(c, DEPTH_U16)
        dbuf[:] = d; cbuf[:] = rgb
        v.integrateDepth(dbuf, p, cbuf, scale)
        other, _, orgb = depth_of(frame(k + 20)[1], DEPTH_U16)
        dbuf[:] = other; cbuf[:] = orgb                       # the call has returned: the buffers are the caller's again
        o.integrate(oracle_cloud(d, scale, rgb, CAM), p)
    check(v, o, "overwritten host buffers")


# ---- reads after depth frames ------------------------------------------------------------------------------------------
def test_reads_equal_a_handle_fed_clouds():
    from tests.test_mesh_incremental_gpu import full_mesh, same
    a, b = engine(CFG_512, True), engine(CFG_512, True)
    inc = pkg.IncrementalMesh(a, 2.0, 1)
    for k in range(0, 10, 2):
        fs = [frame(k), frame(k + 1)]
        ds = [depth_of(c, DEPTH_U16) for _, c in fs]
        a.integrateDepth(ds[0][0], fs[0][0], ds[0][2], 1e-3)
        dd = device([ds[1][0], ds[1][2]])
        a.integrateDepthBatchDevice([dd[0].data_ptr()], [fs[1][0]], depth_format=DEPTH_U16, depth_scale=1e-3, d_rgb_ptrs=[dd[1].data_ptr()])
        for (p, _), (d, scale, rgb) in zip(fs, ds):
            b.integrateCloud(oracle_cloud(d, scale, rgb, CAM), None, p)
        same(inc, a)
    ok(a, a._lib.b200tsdf_sync(a._h)); ok(b, b._lib.b200tsdf_sync(b._h))
    assert_same_nodes(b.download_nodes(), a.download_nodes(), rgb=True)
    pose = frame(3)[0]
    ra, rb = a.renderColoredView(pose, 2), b.renderColoredView(pose, 2)
    for x, y in zip(ra, rb):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    va, ca = full_mesh(a, 2.0, 1)
    vb, cb = full_mesh(b, 2.0, 1)
    assert torch.equal(va.view(torch.int32), vb.view(torch.int32)) and torch.equal(ca, cb)
    na, nb = a.saveDevice(), b.saveDevice()
    assert na == nb
    ba = torch.empty(na, dtype=torch.uint8, device="cuda:0"); bb = torch.empty(nb, dtype=torch.uint8, device="cuda:0")
    a.saveDevice(ba.data_ptr(), na); b.saveDevice(bb.data_ptr(), nb)
    assert torch.equal(ba, bb)
