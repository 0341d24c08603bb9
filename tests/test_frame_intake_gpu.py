"""Every route by which frames reach the device, against the oracle, bit for bit.

Consecutive frames share state across calls: the host numbers every frame (FrameRec::seq), alternates its counter set and
gates its k_front on the previous frame's fold marks when the route publishes them (C == SL, e.g. 512^3 / 3 m with colour).
The numbering must stay in step whichever entry point submits a frame, and a refused call must number nothing.

* Every ordered pair of the nine routes, self-pairs included, on one handle without a sync in between (a de Bruijn walk),
  on a gated grid (with and without the diagnostic counters armed) and on one that is never gated, with the count of gated
  k_front launches.
* Refused calls in the middle of a gated stream: each returns B200TSDF_EINVAL, and the next accepted frame runs gated and
  in step.
* Point layouts (stride, xyz and colour offsets, a misaligned host pointer) through the host routes, packed on the host
  and uploaded as they are.
* Stage schedules of integrateBatchRows: chunk sizes, batch sizes, pack threads and image sizes.
* integrateBatchDevice calls that span several record halves.
* Caller buffers overwritten with another real frame at the earliest moment include/b200tsdf.h allows.
* Image size and packing changes on one handle across resets."""
import ctypes as C
import functools

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle import oracle_py
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256, CFG_512, assert_same_nodes
from tests.test_dynamic_scenes_gpu import debug_timing
from tests.test_edits_gpu import unorganized
from tests.test_pixel_plane_gpu import _repack

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

EINVAL = -1
SEED = 29


def camera(w, h):
    """a camera of w x h pixels with CAM's field of view"""
    f = 525.0 * w / 640
    return synth.Camera(fx=f, fy=f, cx=(w - 1) / 2, cy=(h - 1) / 2, width=w, height=h)


@functools.lru_cache(maxsize=48)
def _frame(k, w, h):
    pose = synth.orbit_pose(synth.S1, 3 * k, 100)
    return pose, synth.make_frame(synth.S1, pose, camera(w, h), color=True, noise_seed=SEED, frame=k, dropout=0.02)


def frame(k, cam=CAM):
    """frame k of the orbit stream seen by cam (a camera() of its size): colour, depth noise and dropout.  Shared: read only."""
    return _frame(k, cam.width, cam.height)


def frames(k0, n, cam=CAM):
    return [frame(k, cam) for k in range(k0, k0 + n)]


def engine(cfg, color, cam=CAM, pool_log2=18):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
    v.setIntegrateColor(color)
    size(v, cam)
    return v


def size(v, cam):
    """setImageSize and the intrinsics of cam, then reset ()"""
    v.setImageSize(cam.width, cam.height)
    v.setCameraIntrinsics(cam.fx, cam.fy, cam.cx, cam.cy)
    v.reset()


def oracle(cfg, color, cam=CAM):
    o = OracleVolume(**dict(cfg, cx=cam.cx, cy=cam.cy), fx=cam.fx, fy=cam.fy, image_width=cam.width,
                     image_height=cam.height, integrate_color=int(color))
    o.reset()
    return o


def organized(pts, cam):
    """the oracle's organise of an unorganised cloud (integrate.cpp:548-607)"""
    return oracle_py.organize(pts, (cam.fx, cam.fy, cam.cx, cam.cy), cam.width, cam.height, rgba_off=16)[0]


def pose_arg(p):
    return np.ascontiguousarray(np.asarray(p, np.float64).reshape(4, 4))


def poses_arg(ps):
    return np.ascontiguousarray(np.stack([pose_arg(p) for p in ps]))


def ok(v, rc, what=""):
    assert rc == 0, f"{what}: {v._lib.b200tsdf_last_error(v._h).decode()} (code {rc})"


def same(v, o, what, *, nodes=None, n_add=None):
    """sync, then the last frame's counts and every node against the oracle (or its stored nodes and count)"""
    ok(v, v._lib.b200tsdf_sync(v._h), what)
    st = v.stats()
    want = o.stats().n_add_observation if n_add is None else n_add
    assert st.n_updates == want, (what, st.n_updates, want)
    try:
        assert_same_nodes(o.dump_nodes() if nodes is None else nodes, v.download_nodes(), rgb=bool(v._cfg.integrate_color))
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None


class HostBuf:
    """a host buffer holding `nbytes` at an address `offset` bytes past a 64-byte boundary; pinned: page-locked memory,
    which the asynchronous uploads read after the call has returned (pageable memory is staged before it returns)"""

    def __init__(self, nbytes, *, offset=0, pinned=False):
        if pinned:
            self._t = torch.empty(nbytes + 128, dtype=torch.uint8, pin_memory=True)
            raw = self._t.numpy()
        else:
            raw = np.empty(nbytes + 128, np.uint8)
        at = (-raw.ctypes.data) % 64 + offset
        self.buf = raw[at:at + nbytes]
        self.addr = self.buf.ctypes.data
        assert self.addr % 64 == offset

    def fill(self, a):
        self.buf[:] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        return self


def host(a, **kw):
    a = np.ascontiguousarray(a)
    return HostBuf(a.nbytes, **kw).fill(a)


def device(arrays):
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()                       # (the engine's streams do not wait for torch's)
    return dev


# ---- the routes ------------------------------------------------------------------------------------------------------
class Routes:
    """the nine integrate routes of one handle.  Each takes [(pose, cloud)] (1 or 2 colour frames, [H, W, 8]) and returns
    what the oracle must integrate for them; buffers that the contract wants alive until the next sync go to `keep`."""

    ONE = ("cloud", "host16", "async_packed", "async_unpacked", "device", "unorg")
    TWO = ("batch_device", "batch_rows", "unorg_batch")
    NAMES = ("cloud", "host16", "async_packed", "async_unpacked", "device", "batch_device", "batch_rows", "unorg", "unorg_batch")

    def __init__(self, v, cam=CAM):
        self.v, self.lib, self.h, self.cam = v, v._lib, v._h, cam
        self.keep = []

    def frames_of(self, name):
        return 2 if name in self.TWO else 1

    def run(self, name, fs):
        assert len(fs) == self.frames_of(name)
        return getattr(self, name)(fs)

    def _host(self, fs, stride, rgba_off, fn, pinned):
        W, H = self.cam.width, self.cam.height
        (p, c), = fs
        b = host(c if stride == 32 else _repack(c, stride, 0, rgba_off), pinned=pinned)
        self.keep.append(b)
        ok(self.v, fn(self.h, C.c_void_p(b.addr), stride, 0, rgba_off, W, H, pose_arg(p).ctypes.data), fn.__name__)
        return fs

    def cloud(self, fs):                           # integrateCloud: 32-byte rows, packed on the host
        (p, c), = fs
        self.v.integrateCloud(c, None, p)
        return fs

    def host16(self, fs):                          # 16-byte rows, colour word at 12: uploaded as they are
        return self._host(fs, 16, 12, self.lib.b200tsdf_integrate, False)

    def async_packed(self, fs):
        return self._host(fs, 32, 16, self.lib.b200tsdf_integrate_async, True)

    def async_unpacked(self, fs):
        return self._host(fs, 16, 12, self.lib.b200tsdf_integrate_async, True)

    def device(self, fs):
        (p, c), = fs
        d, = device([c])
        self.keep.append(d)
        ok(self.v, self.lib.b200tsdf_integrate_device(self.h, C.c_void_p(d.data_ptr()), 32, 0, 16, self.cam.width,
                                                      self.cam.height, pose_arg(p).ctypes.data), "integrate_device")
        return fs

    def batch_device(self, fs):
        dev = device([c for _, c in fs])
        self.keep.append(dev)
        self.v.integrateBatchDevice([d.data_ptr() for d in dev], self.cam.height, self.cam.width, 32, [p for p, _ in fs],
                                    rgba_off=16)
        return fs

    def batch_rows(self, fs):
        bufs = [host(c) for _, c in fs]
        self.keep.append(bufs)
        self.v.integrateBatchRows([b.addr for b in bufs], self.cam.height, self.cam.width, 32, [p for p, _ in fs],
                                  rgba_off=16)
        return fs

    def unorg(self, fs):
        (p, c), = fs
        pts = unorganized(c)
        self.v.integrateUnorganizedCloud(pts, p)
        return [(p, organized(pts, self.cam))]

    def unorg_batch(self, fs):
        pts = [unorganized(c) for _, c in fs]
        dev = device(pts)
        self.keep.append(dev)
        self.v.integrateUnorganizedBatchDevice([d.data_ptr() for d in dev], [len(x) for x in pts], 32, [p for p, _ in fs],
                                               rgba_off=16)
        return [(p, organized(x, self.cam)) for (p, _), x in zip(fs, pts)]


def de_bruijn(k):
    """a cyclic sequence over 0..k-1 in which every ordered pair (a, b), a == b included, occurs exactly once: an Eulerian
    circuit of the complete digraph with loops on k nodes"""
    a, seq = [0] * 3, []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


WALK = [Routes.NAMES[i] for i in de_bruijn(len(Routes.NAMES))]
WALK.append(WALK[0])                                   # 81 pairs, 82 calls


@pytest.mark.parametrize("grid", ["512_colour_gated", "512_colour_gated_uninstrumented", "256_depth"])
def test_every_switch_between_routes(grid):
    """counted: debug_timing arms the diagnostic atomics of k_front and k_celltop_up, so the uninstrumented walk runs the
    kernels as they run in production and checks the nodes only"""
    cfg, color = (CFG_256, False) if grid == "256_depth" else (CFG_512, True)
    counted = grid != "512_colour_gated_uninstrumented"
    assert len(WALK) == 82 and len(set(zip(WALK, WALK[1:]))) == 81
    v, o = engine(cfg, color), oracle(cfg, color)
    r = Routes(v)
    if counted:
        debug_timing(v)                                # arm the k_front counters: [11] gated, [12] waited for the last kernel
    gated = plain = k = 0
    checkpoints = {20, 41, 62, len(WALK)}
    for i, name in enumerate(WALK, 1):
        fs = [frame(j % 45) for j in range(k, k + r.frames_of(name))]
        k += len(fs)
        for p, c in r.run(name, fs):
            o.integrate(c, p)
        if i in checkpoints:
            same(v, o, f"{grid}: call {i} ({name}), frame {k}")
            r.keep.clear()
            if counted:
                d = debug_timing(v)
                gated += int(d[11]); plain += int(d[12])
    # on the gated grid every frame after reset () waits per supercell for its predecessor's fold, whichever route submitted
    # either of them (the first k_front of an unorganised batch is a plain launch behind the organise kernels, but gated too)
    if counted:
        assert (gated, plain) == ((k - 1, 1) if grid == "512_colour_gated" else (0, k)), k


# ---- refused calls -----------------------------------------------------------------------------------------------------
def test_refused_calls_in_a_gated_stream():
    """Each refused call returns B200TSDF_EINVAL and numbers no frame: the accepted frame after it runs gated, the next call
    reports no error (a frame gated on a predecessor that never ran would wait until ERR_FOLD_WAIT), and the volume equals the
    oracle fed the accepted frames only."""
    v, o = engine(CFG_512, True), oracle(CFG_512, True)
    lib, h = v._lib, v._h
    r = Routes(v)
    W, H = CAM.width, CAM.height
    debug_timing(v)
    k = 0
    for name in ("cloud", "device"):
        for p, c in r.run(name, frames(k, 1)):
            o.integrate(c, p)
        k += 1
    ok(v, lib.b200tsdf_sync(h))
    assert tuple(debug_timing(v)[11:13]) == (1, 1)

    p1, c1 = frame(100)
    d1, = device([c1])
    ps40 = poses_arg([p1] * 40)
    pts = unorganized(c1)
    dpts, = device([pts])
    row = host(c1)
    org_opts = pkg.OrganizeOpts(1.0, 0, None)
    ptrs = lambda xs: (C.c_void_p * len(xs))(*xs)
    dp = d1.data_ptr()

    def batch_device(n, xs, w=W, hh=H):
        return lib.b200tsdf_integrate_batch_device(h, n, ptrs(xs), 32, 0, 16, w, hh, ps40.ctypes.data)

    def rows(n, xs, stride=32, xyz_off=0, rgba_off=16, w=W):
        return lib.b200tsdf_integrate_batch_rows(h, n, ptrs(xs), stride, xyz_off, rgba_off, w, H, ps40.ctypes.data)

    def unorg_batch(xs, counts):
        return lib.b200tsdf_integrate_unorganized_batch_device(h, len(xs), ptrs(xs), (C.c_size_t * len(xs))(*counts), 32, 0,
                                                               16, C.byref(org_opts), ps40.ctypes.data)

    def host_call(fn, stride=32, xyz_off=0, rgba_off=16, w=W, hh=H):
        return fn(h, C.c_void_p(row.addr), stride, xyz_off, rgba_off, w, hh, ps40.ctypes.data)

    refusals = [
        ("batch_device null at 1", lambda: batch_device(2, [dp, None])),
        ("batch_device n=40 null at 35", lambda: batch_device(40, [dp] * 35 + [None] + [dp] * 4)),
        ("batch_device wrong width", lambda: batch_device(2, [dp, dp], w=W - 1)),
        ("batch_rows null row", lambda: rows(2, [row.addr, None])),
        ("batch_rows n=33", lambda: rows(33, [row.addr] * 33)),
        ("batch_rows wrong width", lambda: rows(2, [row.addr] * 2, w=W + 1)),
        ("batch_rows bad layout", lambda: rows(2, [row.addr] * 2, rgba_off=30)),
        ("unorg_batch null cloud with points", lambda: unorg_batch([dpts.data_ptr(), None], [len(pts), 5])),
        ("integrate wrong height", lambda: host_call(lib.b200tsdf_integrate, hh=H - 1)),
        ("integrate_device wrong height", lambda: lib.b200tsdf_integrate_device(h, C.c_void_p(dp), 32, 0, 16, W, H + 1,
                                                                                ps40.ctypes.data)),
        ("integrate bad stride", lambda: host_call(lib.b200tsdf_integrate, stride=13)),
        ("integrate_async bad xyz_off", lambda: host_call(lib.b200tsdf_integrate_async, xyz_off=2)),
        ("integrate_async rgba past the point", lambda: host_call(lib.b200tsdf_integrate_async, rgba_off=32)),
        ("integrate_unorganized bad layout", lambda: lib.b200tsdf_integrate_unorganized(
            h, C.c_void_p(pts.ctypes.data), len(pts), 32, 0, 6, C.byref(org_opts), ps40.ctypes.data)),
    ]
    accept = ("batch_device", "cloud", "device", "batch_rows", "unorg_batch", "async_unpacked", "unorg", "host16")
    for i, (what, refuse) in enumerate(refusals):
        assert refuse() == EINVAL, what
        name = accept[i % len(accept)]
        fs = frames(k, r.frames_of(name))
        k += len(fs)
        for p, c in r.run(name, fs):
            o.integrate(c, p)
        ok(v, lib.b200tsdf_sync(h), f"after {what}")
        r.keep.clear()
        assert tuple(debug_timing(v)[11:13]) == (len(fs), 0), what
    same(v, o, "after every refusal")
    del d1, dpts


# ---- point layouts through the host routes ---------------------------------------------------------------------------
LAYOUTS = {
    # name: (stride, xyz_off, rgba_off, host address offset)
    "xyz12": (12, 0, -1, 0),
    "xyzc16": (16, 0, 12, 0),
    "xyz20_at8": (20, 8, -1, 0),
    "stride24_scalar": (24, 0, 16, 0),
    "pcl32_sse": (32, 0, 16, 0),
    "pcl32_misaligned": (32, 0, 16, 4),
    "stride48": (48, 8, 40, 0),
    "rgba_before_xyz": (32, 16, 0, 0),
}
NLAYOUT = 3
_ORACLE = {}
_LAYOUT_ENGINES = {}


def layout_engine(color, host_pack, monkeypatch):
    """one handle per (colour, B200TSDF_HOST_PACK), which b200tsdf_create reads; reset () between the layouts"""
    key = (color, host_pack)
    if key in _LAYOUT_ENGINES:
        _LAYOUT_ENGINES[key].reset()
    else:
        if host_pack is not None:
            monkeypatch.setenv("B200TSDF_HOST_PACK", host_pack)
        _LAYOUT_ENGINES[key] = engine(CFG_512, color)
    return _LAYOUT_ENGINES[key]


def oracle_run(key, cfg, color, fs, feed=lambda c: c):
    """nodes and last-frame count of the oracle fed fs, once per key"""
    if key not in _ORACLE:
        o = oracle(cfg, color, camera(fs[0][1].shape[1], fs[0][1].shape[0]))
        for p, c in fs:
            o.integrate(feed(c), p)
        _ORACLE[key] = (o.dump_nodes(), o.stats().n_add_observation)
    return _ORACLE[key]


def fuse_layout(v, route, fs, stride, xyz_off, rgba_off, offset):
    lib, h = v._lib, v._h
    W, H = CAM.width, CAM.height
    bufs = [host(_repack(c, stride, xyz_off, rgba_off), offset=offset, pinned=route == "async") for _, c in fs]
    if route in ("integrate", "async"):
        fn = lib.b200tsdf_integrate if route == "integrate" else lib.b200tsdf_integrate_async
        for b, (p, _) in zip(bufs, fs):
            ok(v, fn(h, C.c_void_p(b.addr), stride, xyz_off, rgba_off, W, H, pose_arg(p).ctypes.data), route)
    else:
        for lo, hi in ((0, 1), (1, len(fs))):
            arr = (C.c_void_p * (hi - lo))(*[b.addr for b in bufs[lo:hi]])
            ps = poses_arg([p for p, _ in fs[lo:hi]])
            ok(v, lib.b200tsdf_integrate_batch_rows(h, hi - lo, arr, stride, xyz_off, rgba_off, W, H, ps.ctypes.data), route)
    ok(v, lib.b200tsdf_sync(h), route)
    return bufs


# B200TSDF_HOST_PACK applies to points wider than 16 bytes only: those run with it at 1 and at 0
LAYOUT_RUNS = [(name, route, hp) for name, (stride, _, _, _) in LAYOUTS.items() for route in ("integrate", "async", "rows")
               for hp in (("1", "0") if stride > 16 else (None,))]


@pytest.mark.parametrize("layout,route,host_pack", LAYOUT_RUNS)
def test_point_layouts_through_the_host_routes(layout, route, host_pack, monkeypatch):
    """b200tsdf_integrate / _integrate_async / _integrate_batch_rows in every layout, against a colour volume and a depth-only
    one (which ignores the colour bytes); points wider than 16 bytes both packed on the host and uploaded as they are"""
    stride, xyz_off, rgba_off, offset = LAYOUTS[layout]
    fs = frames(200, NLAYOUT)
    for color in (True, False):
        # a colour volume fed points without colour bytes takes colour word 0, as the oracle does for [H, W, 4] clouds
        key = ("layout", color, color and rgba_off >= 0)
        nodes, n_add = oracle_run(key, CFG_512, color, fs, (lambda c: c) if rgba_off >= 0 or not color else (lambda c: c[..., :4]))
        v = layout_engine(color, host_pack, monkeypatch)
        fuse_layout(v, route, fs, stride, xyz_off, rgba_off, offset)
        same(v, None, f"{layout} {route} HOST_PACK={host_pack} colour={color}", nodes=nodes, n_add=n_add)


# ---- stage schedules of integrateBatchRows -----------------------------------------------------------------------------
ROWS_CASES = {
    # id: (B200TSDF_ROWS_CHUNK, B200TSDF_PACK_THREADS, B200TSDF_HOST_PACK, image size, debug_flags)
    "chunk1": ("1", None, None, (640, 480), 0),
    "chunk2_threads1": ("2", "1", None, (640, 480), 0),
    "chunk3_threads3": ("3", "3", None, (640, 480), 0),
    "chunk5": ("5", None, None, (640, 480), 0),
    "chunk32_threads1": ("32", "1", None, (640, 480), 0),
    "chunk5_unpacked": ("5", None, "0", (640, 480), 0),
    "default_64x48_threads3": (None, "3", None, (64, 48), 0),
    "default_64x48_threads3_general": (None, "3", None, (64, 48), 1),
    "chunk3_643x479_threads1": ("3", "1", None, (643, 479), 0),
}
ROWS_SIZES = (3, 32, 0, 1, 7, 2)                     # 45 frames; both buffer sets see several batch sizes
# Measured on an H100, on every run: at 64x48 on the supercell route of 512^3 / 3 m (k_celltop_down / k_bricks / k_celltop_up)
# the 32-frame call leaves 9 nodes at levels 4-5 (the tier-1 brick) with {sdf, weight} other than the oracle's, the same 9
# through integrateBatchDevice, and with the per-supercell gate of k_front off as well.  The same batches through the per-level
# sweeps (debug_flags bit 1) and through the general kernel (bit 0, the _general case) are bit-exact.  Strict: the case fails
# once the divergence is fixed, and the mark must go then.
SMALL_FRAMES_SUPERCELL = pytest.mark.xfail(reason="supercell route: 9 tier-1 nodes of the 64x48 stream differ from the oracle",
                                           strict=True)


@pytest.mark.parametrize("case", [pytest.param(c, marks=SMALL_FRAMES_SUPERCELL) if c == "default_64x48_threads3" else c
                                  for c in ROWS_CASES])
def test_rows_stage_schedules(case, monkeypatch):
    chunk, threads, hpack, (w, hh), flags = ROWS_CASES[case]
    for var, val in (("B200TSDF_ROWS_CHUNK", chunk), ("B200TSDF_PACK_THREADS", threads), ("B200TSDF_HOST_PACK", hpack)):
        if val is not None:
            monkeypatch.setenv(var, val)
    cam = camera(w, hh)
    fs = frames(300, sum(ROWS_SIZES), cam)
    nodes, n_add = oracle_run(("rows", w, hh), CFG_512, True, fs)
    v = engine(CFG_512, True, cam)
    if flags:
        v._cfg.debug_flags = flags
        v._push()
        v.reset()
    keep, at = [], 0
    for n in ROWS_SIZES:
        if n == 0:
            before = v.stats().n_updates
            ok(v, v._lib.b200tsdf_integrate_batch_rows(v._h, 0, None, 32, 0, 16, w, hh, None), "n == 0")
            assert v.stats().n_updates == before
            continue
        part = fs[at:at + n]
        at += n
        bb = [host(c) for _, c in part]
        keep = (keep + [bb])[-2:]                      # (the unpacked upload may read them until two further calls)
        v.integrateBatchRows([b.addr for b in bb], hh, w, 32, [p for p, _ in part], rgba_off=16)
    same(v, None, case, nodes=nodes, n_add=n_add)


# ---- integrateBatchDevice across record halves -------------------------------------------------------------------------
def test_batch_device_across_record_halves():
    """calls of 33, 64 and 65 frames (several record halves each, halves of different sizes replaying cached graphs), then
    1 and 31, on one handle"""
    cam = camera(320, 240)
    sizes = (33, 64, 65, 1, 31)
    fs = frames(400, sum(sizes), cam)
    v, o = engine(CFG_512, True, cam), oracle(CFG_512, True, cam)
    dev = device([c for _, c in fs])
    at = 0
    for n in sizes:
        part = slice(at, at + n)
        at += n
        v.integrateBatchDevice([d.data_ptr() for d in dev[part]], cam.height, cam.width, 32, [p for p, _ in fs[part]],
                               rgba_off=16)
        for p, c in fs[part]:
            o.integrate(c, p)
        same(v, o, f"after the call of {n} frames")
    del dev


# ---- caller-buffer lifetime --------------------------------------------------------------------------------------------
NLIFE = 8
LIFETIME = {
    # id: (entry point, stride, B200TSDF_HOST_PACK, calls after which a call's buffers may be rewritten)
    "integrate_unpacked": ("integrate", 16, None, 0),
    "integrate_packed": ("integrate", 32, None, 0),
    "async_packed": ("async", 32, None, 0),
    "async_unpacked": ("async", 16, None, 2),
    "rows_packed": ("rows", 32, None, 0),
    "rows_unpacked": ("rows", 32, "0", 2),
}


@pytest.mark.parametrize("case", list(LIFETIME))
def test_buffers_rewritten_as_soon_as_the_contract_allows(case, monkeypatch):
    """Each buffer (page-locked) is overwritten with another real frame's points at the earliest moment include/b200tsdf.h
    allows; the volume must equal the oracle fed the frames as they were.  A pass does not prove the absence of a race, a
    failure is a violation."""
    entry, stride, hpack, later = LIFETIME[case]
    if hpack is not None:
        monkeypatch.setenv("B200TSDF_HOST_PACK", hpack)
    fs = frames(500, NLIFE)
    decoys = [c for _, c in frames(550, NLIFE)]
    nodes, n_add = oracle_run(("life",), CFG_512, True, fs)
    v = engine(CFG_512, True)
    lib, h = v._lib, v._h
    lay = lambda c: c if stride == 32 else _repack(c, 16, 0, 12)
    rgba = 16 if stride == 32 else 12
    per_call = 2 if entry == "rows" else 1
    calls = [list(range(i, i + per_call)) for i in range(0, NLIFE, per_call)]
    bufs = [host(lay(c), pinned=True) for _, c in fs]
    for j, idx in enumerate(calls):
        if entry == "rows":
            arr = (C.c_void_p * len(idx))(*[bufs[i].addr for i in idx])
            ok(v, lib.b200tsdf_integrate_batch_rows(h, len(idx), arr, stride, 0, rgba, CAM.width, CAM.height,
                                                     poses_arg([fs[i][0] for i in idx]).ctypes.data), case)
        else:
            fn = lib.b200tsdf_integrate if entry == "integrate" else lib.b200tsdf_integrate_async
            i, = idx
            ok(v, fn(h, C.c_void_p(bufs[i].addr), stride, 0, rgba, CAM.width, CAM.height, pose_arg(fs[i][0]).ctypes.data), case)
        if j >= later:
            for i in calls[j - later]:
                bufs[i].fill(lay(decoys[i]))
    same(v, None, case, nodes=nodes, n_add=n_add)


# ---- image size and packing changes on one handle --------------------------------------------------------------------
def test_image_size_and_packing_changes_on_one_handle():
    """reset () at 320x240, 640x480, 643x479 and 320x240 again; at each size frames go through the host, asynchronous, row and
    unorganised routes, unpacked first and packed after (the packed staging is allocated mid-stream), without a sync"""
    v = engine(CFG_512, True, camera(320, 240))
    seq = ("host16", "async_unpacked", "cloud", "async_packed", "batch_rows", "unorg", "host16", "batch_rows16", "cloud")
    for s, (w, hh) in enumerate(((320, 240), (640, 480), (643, 479), (320, 240))):
        cam = camera(w, hh)
        if s:
            size(v, cam)
        o = oracle(CFG_512, True, cam)
        r = Routes(v, cam)
        k = 600 + 20 * s
        for name in seq:
            if name == "batch_rows16":                 # 16-byte rows: uploaded as they are and fused where they landed
                fs = frames(k, 2, cam)
                bufs = [host(_repack(c, 16, 0, 12)) for _, c in fs]
                r.keep.append(bufs)
                v.integrateBatchRows([b.addr for b in bufs], hh, w, 16, [p for p, _ in fs], rgba_off=12)
            else:
                fs = frames(k, r.frames_of(name), cam)
                fs = r.run(name, fs)
            k += len(fs)
            for p, c in fs:
                o.integrate(c, p)
        same(v, o, f"segment {s} at {w}x{hh}")
        r.keep.clear()
