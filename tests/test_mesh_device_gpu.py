"""Marching cubes and the mesh post-processing into device memory: reconstructDevice, flattenVerticesDevice and
cleanupMeshDevice, bit for bit against the host entry points.

* Same mesh as reconstruct(): colour modes 0/1/2 x w_min 0, 2 and 2.5 on the 256^3 colour stream (a C > SL shape, also
  compared with the restatement), RGBNormalized (K3), the 2048^3 / 10 m case K4, a 128^3 / 3 m volume, a non-identity
  global transform, a volume from load() and an empty volume.
* Buffer protocol: count query, exact and larger capacities, a capacity too small, no colour buffer, misalignment, ESTATE.
* Ordering: integrateBatchDevice followed by reconstructDevice with no sync in between meshes the fused volume.
* flatten / cleanup on device arrays equal the host entry points, in soup mode and with indices, the inputs unchanged and
  nothing written past the results; every refusal leaves the outputs untouched.
* The whole back end in device memory equals reconstruct -> flattenVertices -> cleanupMesh."""

import ctypes as C

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests import dynamic_cases
from tests.common import CFG_256, frames
from tests.test_meshpost import adversarial_mesh, mc_soup, scattered_faces

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FBADBAD
RGB_SENTINEL = 0xA5
MODES = [(cm, w) for cm in (0, 1, 2) for w in (0.0, 2.0, 2.5)]
GT = np.array([[0.0, -0.8, 0.6, 0.25], [1.0, 0.0, 0.0, -1.5], [0.0, 0.6, 0.8, 3.0], [0, 0, 0, 1]])


def _engine(cfg, pool_log2=18, **extra):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    for k, x in {**cfg, **extra}.items():
        setattr(v._cfg, k, x)
    v._push()
    v.reset()
    return v


def _stream256(**extra):
    v = _engine(CFG_256, integrate_color=1, **extra)
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        v.integrateCloud(cloud, None, pose)
    return v


def _case(cid):
    case = dynamic_cases.CASES[cid]
    v = _engine(case.config())
    for pose, cloud in case.frames():
        v.integrateCloud(cloud, None, pose)
    return v


def _build(name, tmp_path_factory):
    if name == "stream256":
        return _stream256()
    if name in ("K3", "K4"):
        return _case(name)
    if name == "128^3":
        v = _engine(dict(CFG_256, xres=128, yres=128, zres=128), integrate_color=1)
        for pose, cloud in frames(synth.S1, 4, stride=9, color=True, noise_seed=7):
            v.integrateCloud(cloud, None, pose)
        return v
    if name == "transform":
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
        for k, x in dict(CFG_256, integrate_color=1).items():
            setattr(v._cfg, k, x)
        v.setGlobalTransform(GT)
        v.reset()
        for pose, cloud in frames(synth.S1, 3, stride=11, color=True, noise_seed=9):
            v.integrateCloud(cloud, None, pose)
        return v
    if name == "loaded":
        src = _engine(CFG_256, integrate_color=1)
        for pose, cloud in frames(synth.S1, 3, stride=13, color=True, noise_seed=3):
            src.integrateCloud(cloud, None, pose)
        path = str(tmp_path_factory.mktemp("vol") / "v.vol")
        src.save(path)
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
        v.load(path)
        return v
    assert name == "empty"
    return _engine(CFG_256)


VOLUMES = ["stream256", "K3", "K4", "128^3", "transform", "loaded", "empty"]


@pytest.fixture(scope="module")
def volumes(tmp_path_factory):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _build(name, tmp_path_factory)
            cache[name].sync()
        return cache[name]
    return get


def _mc(vol, cm=0, wmin=0.0):
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(vol)
    mc.setMinWeight(wmin); mc.setColorByRGB(cm == 1); mc.setColorByConfidence(cm == 2)
    return mc


def device_mesh(mc, capacity=None, pad=5, rgb=True):
    """a count query, then reconstructDevice into torch buffers of capacity + pad vertices pre-filled with the sentinels:
    (count, vertex words [capacity + pad, 3] uint32, colours [capacity + pad, 3] uint8 or None)"""
    import torch
    n = mc.reconstructDevice()
    cap = n if capacity is None else capacity
    dv = torch.full(((cap + pad) * 3,), SENTINEL, dtype=torch.int32, device="cuda")
    dc = torch.full(((cap + pad) * 3,), RGB_SENTINEL, dtype=torch.uint8, device="cuda") if rgb else None
    torch.cuda.synchronize()
    assert mc.reconstructDevice(dv.data_ptr(), cap, None if dc is None else dc.data_ptr()) == n
    return n, dv.cpu().numpy().view(np.uint32).reshape(-1, 3), None if dc is None else dc.cpu().numpy().reshape(-1, 3)


def assert_same_mesh(n, words, cols, verts, rgb):
    """the device result (device_mesh) equals reconstruct()'s arrays bit for bit, and nothing past them was written"""
    assert n == len(verts)
    assert np.array_equal(words[:n], verts.view(np.uint32)) and (words[n:] == SENTINEL).all()
    if cols is not None:
        if rgb is None:
            assert (cols == RGB_SENTINEL).all()
        else:
            assert np.array_equal(cols[:n], rgb) and (cols[n:] == RGB_SENTINEL).all()


@pytest.mark.parametrize("cm,wmin", MODES)
@pytest.mark.parametrize("name", VOLUMES)
def test_device_mesh_equals_host_mesh(volumes, name, cm, wmin):
    vol = volumes(name)
    mc = _mc(vol, cm, wmin)
    verts, rgb, polys = mc.reconstruct()
    n, words, cols = device_mesh(mc)
    assert_same_mesh(n, words, cols, verts, rgb)
    assert (rgb is None) == (cm == 0) or n == 0
    if name == "empty":
        assert n == 0
    elif wmin == 0.0:
        assert n > 3000


def test_device_mesh_equals_restatement():
    o = OracleVolume(**CFG_256, integrate_color=1)
    o.reset()
    for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
        o.integrate(cloud, pose)
    vol = _stream256()
    for cm, wmin in ((0, 2.0), (1, 0.0), (2, 2.5)):
        n, words, cols = device_mesh(_mc(vol, cm, wmin))
        va, ca = o.mesh(wmin, cm)
        assert n == len(va) > 3000
        assert np.array_equal(words[:n], np.asarray(va, np.float32).reshape(-1, 3).view(np.uint32))
        if cm:
            assert np.array_equal(cols[:n], np.asarray(ca).reshape(-1, 3))


def _code(fn):
    with pytest.raises(pkg.B200Error) as e:
        fn()
    return str(e.value).rsplit("(code ", 1)[1].rstrip(")")


def test_buffer_protocol(volumes):
    import torch
    vol = volumes("stream256")
    mc = _mc(vol, 1, 0.0)
    verts, rgb, _ = mc.reconstruct()
    n = len(verts)
    assert n > 3000 and n % 3 == 0
    # count only: nothing is written, not even into a colour buffer that is passed
    dc = torch.full((n * 3,), RGB_SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert mc.reconstructDevice(None, 0, dc.data_ptr()) == n
    assert (dc.cpu().numpy() == RGB_SENTINEL).all()
    # exact capacity; a larger one leaves the sentinels past 12 n / 3 n bytes
    assert_same_mesh(*device_mesh(mc, capacity=n, pad=0), verts, rgb)
    assert_same_mesh(*device_mesh(mc, capacity=n + 100, pad=3), verts, rgb)
    # capacity n - 3: EINVAL, the count is reported, nothing is written
    dv = torch.full((n * 3,), SENTINEL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    cnt = C.c_size_t(0)
    rc = vol._lib.b200tsdf_mesh_device(vol._h, 0.0, 1, C.c_void_p(dv.data_ptr()), C.c_void_p(dc.data_ptr()), n - 3, C.byref(cnt))
    assert rc == -1 and cnt.value == n
    assert (dv.cpu().numpy().view(np.uint32) == SENTINEL).all() and (dc.cpu().numpy() == RGB_SENTINEL).all()
    assert _code(lambda: mc.reconstructDevice(dv.data_ptr(), n - 3, dc.data_ptr())) == "-1"
    # a colour mode without a colour buffer: the vertices only
    nn, words, _ = device_mesh(mc, rgb=False)
    assert_same_mesh(nn, words, None, verts, rgb)
    # misaligned vertices
    assert _code(lambda: mc.reconstructDevice(dv.data_ptr() + 2, n, None)) == "-1"
    # before reset()
    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    assert _code(lambda: _mc(fresh).reconstructDevice(dv.data_ptr(), n, None)) == "-5"
    assert _code(lambda: _mc(fresh).reconstructDevice()) == "-5"
    assert mc.reconstructDevice() == n                                               # the handle still works


def test_mesh_is_stream_ordered_after_integrate():
    import torch
    stream = list(frames(synth.S1, 32, stride=3, color=True, noise_seed=21))
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in stream]
    torch.cuda.synchronize()
    H, W = dev[0].shape[:2]
    v = _engine(CFG_256, integrate_color=1)
    v.integrateBatchDevice([d.data_ptr() for d in dev], H, W, 32, [p for p, _ in stream], rgba_off=16)
    mc = _mc(v, 1, 0.0)
    n, words, cols = device_mesh(mc)                                                  # no sync before the count query
    ref = _engine(CFG_256, integrate_color=1)
    for pose, cloud in stream:
        ref.integrateCloud(cloud, None, pose)
    verts, rgb, _ = _mc(ref, 1, 0.0).reconstruct()
    assert n > 3000
    assert_same_mesh(n, words, cols, verts, rgb)


# ---- mesh post-processing ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def post_vol():
    return _engine(CFG_256, pool_log2=12)


@pytest.fixture(scope="module")
def soup():
    return mc_soup()


def _device_post(fn, vol, v, t, soup_mode, *args):
    """fn on device copies of (v, t) into outputs sized like the inputs plus a margin, all pre-filled with SENTINEL; checks
    that the inputs are byte-identical afterwards and that nothing was written past the result.  -> (verts, tris)"""
    import torch
    pad = 7
    dv = torch.from_numpy(np.ascontiguousarray(v, np.float32).reshape(-1)).cuda()
    dt = torch.from_numpy(np.ascontiguousarray(t, np.int32).reshape(-1)).cuda()
    ov = torch.full((3 * len(v) + pad,), SENTINEL, dtype=torch.int32, device="cuda")
    ot = torch.full((3 * len(t) + pad,), SENTINEL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    try:
        nv, nt = fn(vol, dv.data_ptr() if len(v) else None, len(v), None if soup_mode else dt.data_ptr(), len(t),
                    ov.data_ptr(), ot.data_ptr(), *args)
    finally:
        assert np.array_equal(dv.cpu().numpy().view(np.uint32), np.asarray(v, np.float32).reshape(-1).view(np.uint32))
        assert np.array_equal(dt.cpu().numpy(), np.asarray(t, np.int32).reshape(-1))
    ov, ot = ov.cpu().numpy(), ot.cpu().numpy()
    assert (ov[3 * nv:].view(np.uint32) == SENTINEL).all() and (ot[3 * nt:].view(np.uint32) == SENTINEL).all()
    return ov[:3 * nv].view(np.float32).reshape(-1, 3), ot[:3 * nt].reshape(-1, 3)


def same(a, b):
    return a[0].shape == b[0].shape and a[1].shape == b[1].shape and np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) \
        and np.array_equal(a[1], b[1])


def _meshes(soup):
    return {"soup": soup, "adversarial": adversarial_mesh(1), "scattered": scattered_faces(5, *soup),
            "empty": (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))}


@pytest.mark.parametrize("mesh", ["soup", "adversarial", "scattered", "empty"])
def test_flatten_device_equals_host(post_vol, soup, mesh):
    v, t = _meshes(soup)[mesh]
    for r in (0.0001, 0.0, -1.0, float("nan"), 0.003):
        want = pkg.flattenVertices(v, t, r)
        for soup_mode in ((False, True) if mesh in ("soup", "empty") else (False,)):
            got = _device_post(pkg.flattenVerticesDevice, post_vol, v, t, soup_mode, r)
            assert same(want, got), (mesh, r, soup_mode)
    if mesh == "soup":
        assert len(pkg.flattenVertices(v, t)[0]) < len(v) / 2


@pytest.mark.parametrize("mesh", ["soup", "adversarial", "scattered", "empty"])
def test_cleanup_device_equals_host(post_vol, soup, mesh):
    v, t = _meshes(soup)[mesh]
    for d in (0.02, 0.0, -1.0, float("nan"), 0.005):
        for k in (1, 3, 5, 16):
            want = pkg.cleanupMesh(v, t, d, k)
            for soup_mode in ((False, True) if mesh in ("soup", "empty") else (False,)):
                got = _device_post(pkg.cleanupMeshDevice, post_vol, v, t, soup_mode, d, k)
                assert same(want, got), (mesh, d, k, soup_mode)


def test_post_processing_refusals_leave_outputs_untouched(post_vol, soup):
    import torch
    v, t = scattered_faces(5, *soup)
    t_hi, t_neg = t.copy(), t.copy()
    t_hi[len(t) // 2, 1] = len(v)
    t_neg[len(t) - 1, 2] = -1

    def refused(fn, v, t, soup_mode, *args):
        """fn on device copies of (v, t) into SENTINEL-filled outputs sized like the inputs plus a margin: the B200 error code,
        after checking that neither an output nor an input byte changed"""
        pad = 7
        dv = torch.from_numpy(np.ascontiguousarray(v, np.float32).reshape(-1)).cuda()
        dt = torch.from_numpy(np.ascontiguousarray(t, np.int32).reshape(-1)).cuda()
        ov = torch.full((3 * len(v) + pad,), SENTINEL, dtype=torch.int32, device="cuda")
        ot = torch.full((3 * len(t) + pad,), SENTINEL, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        code = _code(lambda: fn(post_vol, dv.data_ptr(), len(v), None if soup_mode else dt.data_ptr(), len(t),
                                ov.data_ptr(), ot.data_ptr(), *args))
        assert (ov.cpu().numpy().view(np.uint32) == SENTINEL).all() and (ot.cpu().numpy().view(np.uint32) == SENTINEL).all()
        assert np.array_equal(dv.cpu().numpy().view(np.uint32), np.asarray(v, np.float32).reshape(-1).view(np.uint32))
        assert np.array_equal(dt.cpu().numpy(), np.asarray(t, np.int32).reshape(-1))
        return code

    for fn, args in ((pkg.flattenVerticesDevice, (0.0001,)), (pkg.cleanupMeshDevice, (0.02, 5))):
        for bad in (t_hi, t_neg):                                                        # found on the device
            assert refused(fn, v, bad, False, *args) == "-1"
        sv, st = soup
        assert refused(fn, sv, st[:-1], True, *args) == "-1"                             # nverts != 3 * ntris
    assert refused(pkg.cleanupMeshDevice, v, t, False, 0.02, 17) == "-1"
    assert refused(pkg.cleanupMeshDevice, v, t, False, 0.02, 0) == "-1"
    # outputs overlapping an input
    dv = torch.from_numpy(v.reshape(-1)).cuda(); dt = torch.from_numpy(t.reshape(-1)).cuda()
    ov = torch.full((3 * len(v),), SENTINEL, dtype=torch.int32, device="cuda")
    ot = torch.full((3 * len(t),), SENTINEL, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    for fn, args in ((pkg.flattenVerticesDevice, (0.0001,)), (pkg.cleanupMeshDevice, (0.02, 5))):
        for o_v, o_t in ((dv.data_ptr(), ot.data_ptr()), (ov.data_ptr(), dt.data_ptr()), (ov.data_ptr(), dv.data_ptr() + 4),
                         (dt.data_ptr() + 12 * (len(t) - 1), ot.data_ptr())):
            assert _code(lambda: fn(post_vol, dv.data_ptr(), len(v), dt.data_ptr(), len(t), o_v, o_t, *args)) == "-1"
    assert np.array_equal(dv.cpu().numpy(), v.reshape(-1)) and np.array_equal(dt.cpu().numpy(), t.reshape(-1))
    assert (ov.cpu().numpy().view(np.uint32) == SENTINEL).all() and (ot.cpu().numpy().view(np.uint32) == SENTINEL).all()
    fresh = pkg.TSDFVolumeOctree(device=0, pool_log2=12)
    assert _code(lambda: pkg.flattenVerticesDevice(fresh, dv.data_ptr(), len(v), dt.data_ptr(), len(t), ov.data_ptr(), ot.data_ptr())) == "-5"
    assert _code(lambda: pkg.cleanupMeshDevice(fresh, dv.data_ptr(), len(v), dt.data_ptr(), len(t), ov.data_ptr(), ot.data_ptr())) == "-5"
    assert same(pkg.flattenVertices(v, t), _device_post(pkg.flattenVerticesDevice, post_vol, v, t, False, 0.0001))   # still works


@pytest.mark.parametrize("name", ["stream256", "K4"])
def test_whole_back_end_in_device_memory(volumes, name):
    import torch
    vol = volumes(name)
    mc = _mc(vol, 0, 0.0)
    verts, _, polys = mc.reconstruct()
    want = pkg.cleanupMesh(*pkg.flattenVertices(verts, polys))
    n = mc.reconstructDevice()
    assert n > 3000
    d_v = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    f_v = torch.empty((n, 3), dtype=torch.float32, device="cuda"); f_t = torch.empty((n // 3, 3), dtype=torch.int32, device="cuda")
    c_v = torch.empty((n, 3), dtype=torch.float32, device="cuda"); c_t = torch.empty((n // 3, 3), dtype=torch.int32, device="cuda")
    assert mc.reconstructDevice(d_v.data_ptr(), n) == n
    nv, nt = pkg.flattenVerticesDevice(vol, d_v.data_ptr(), n, None, n // 3, f_v.data_ptr(), f_t.data_ptr())
    nv, nt = pkg.cleanupMeshDevice(vol, f_v.data_ptr(), nv, f_t.data_ptr(), nt, c_v.data_ptr(), c_t.data_ptr())
    got = (c_v[:nv].cpu().numpy(), c_t[:nt].cpu().numpy())
    assert same(want, got) and nt > 1000
