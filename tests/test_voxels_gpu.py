"""getContainingVoxel (k_voxels) and the dense crop (k_dense) of the CUDA engine against the C++ restatement
(oracle/tsdf_oracle_voxels.cpp) and the digests of the reference's own octree_->getContainingVoxel (tests/golden/voxel_pins.json):
every field bit for bit.  Outputs go into sentinel-filled buffers with guard bytes, and no byte outside the extent may change."""
import importlib.util
import json
import os

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from oracle.voxels_py import VoxelsOracleVolume
from tests import voxels
from tests.common import CAM, CFG_256

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_voxel_pins", os.path.join(ROOT, "tools", "make_voxel_pins.py"))
mvp = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mvp)
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "voxel_pins.json")))
EINVAL, ESTATE = -1, -5
GUARD = 4096                                    # bytes of sentinel after every output's extent
SENTINEL = 0xA5


def engine(cfg, pool_log2=18, **kw):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, **kw)
    for k, x in cfg.items():
        setattr(v._cfg, k, x)
    v._push()
    v.reset()
    return v


class Fused:
    """the engine and the restatement after the same frames"""

    def __init__(self, cfg, frames, pool_log2=18):
        self.v = engine(cfg, pool_log2)
        self.o = VoxelsOracleVolume(**cfg)
        self.o.reset()
        for pose, cloud in frames:
            self.v.integrateCloud(cloud, None, pose)
            self.o.integrate(cloud, pose)
        self.size, self.res = cfg["xsize"], cfg["xres"]


def guarded(nbytes):
    t = torch.full((nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device="cuda")
    return t


def dense_engine(v, box, outputs=("d", "w", "rgb", "level")):
    """extractDenseDevice into sentinel-filled buffers; checks the guard bytes and returns the outputs as numpy arrays"""
    shape = tuple(int(box[a + 3] - box[a]) for a in range(3))
    n = int(np.prod(shape))
    spec = {"d": (4, np.float32, shape), "w": (4, np.float32, shape), "rgb": (3, np.uint8, shape + (3,)), "level": (1, np.int8, shape)}
    bufs = {k: guarded(n * spec[k][0]) for k in outputs}
    v.extractDenseDevice(box, **{f"d_{k}": b.data_ptr() for k, b in bufs.items()})
    v.sync()
    out = {}
    for k, b in bufs.items():
        host = b.cpu().numpy()
        assert (host[n * spec[k][0]:] == SENTINEL).all(), f"{k}: a byte past the extent changed"
        out[k] = host[:n * spec[k][0]].view(spec[k][1]).reshape(spec[k][2])
    return out


def lookups_engine(v, pts, min_size=-1.0):
    """the host entry point and the device entry point (into a guarded buffer) must agree; returns the records"""
    host = v.getContainingVoxels(pts, min_size)
    n = len(host)
    if n:
        x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)).cuda()
        b = guarded(44 * n)
        v.getContainingVoxelsDevice(x.data_ptr(), n, b.data_ptr(), min_size)
        v.sync()
        h = b.cpu().numpy()
        assert (h[44 * n:] == SENTINEL).all()
        assert h[:44 * n].tobytes() == host.tobytes()
    return host


def outputs_engine(v, case):
    return mvp.outputs(lambda p, ms=-1.0: lookups_engine(v, p, ms), case)


def assert_same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), k


# ---- the pinned cases: lookups and crops equal the reference's digests and the restatement ---------------------------------
@pytest.mark.parametrize("name", sorted(mvp.CASES))
def test_pinned_cases(name):
    case = mvp.CASES[name]
    cfg = dict(case[0], **mvp.color_kw(case[4]))
    v = engine(cfg)
    mvp.fuse(v_adapter(v), case)
    got = outputs_engine(v, case)
    assert mvp.digests(got) == PINS["cases"][name]
    for b in mvp.BOXES[cfg["xres"]]:                                   # k_dense, each output, against the lookups it restates
        dense = dense_engine(v, b)
        for k, a in dense.items():
            assert a.tobytes() == got[f"dense{list(b)}.{k}"].tobytes(), (b, k)


class v_adapter:
    def __init__(self, v):
        self.v = v

    def integrate(self, cloud, pose):
        self.v.integrateCloud(cloud, None, pose)


# ---- every shape of tests/test_leaves_gpu.py, K1 / K4 / K5 after carving, a loaded volume ------------------------------------
def _shape(res, size, cell):
    return dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy,
                max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)


SHAPES = {
    "128_3.0_0.5": (_shape(128, 3.0, 0.5), "shape", 2, 6, None, 9, 0.0),
    "1024_3.0_0.5": (_shape(1024, 3.0, 0.5), "shape", 2, 6, None, 9, 0.0),
    "256_2.7_0.3": (_shape(256, 2.7, 0.3), "shape", 2, 6, "RGB", 9, 0.0),
    "512_12.0_0.5": (_shape(512, 12.0, 0.5), "shape", 2, 6, None, 9, 0.0),
    "256": (CFG_256, "S1", 3, 9, "RGB", 5, 0.0),
    "512": (dict(CFG_256, xres=512, yres=512, zres=512), "S1", 3, 9, "RGBNormalized", 5, 0.0),
    "2048_10.0": (dict(CFG_256, xres=2048, yres=2048, zres=2048, xsize=10.0, ysize=10.0, zsize=10.0), "S2", 2, 5, "RGB", 5, 0.0),
}
CROPS = {128: [(5, 60, 33, 70, 128, 41)], 256: [(17, 100, 3, 18, 200, 256)], 512: [(301, 7, 250, 345, 70, 291)],
         1024: [(500, 480, 530, 547, 513, 560), (1016, 1000, 1020, 1024, 1024, 1024)],
         2048: [(1001, 998, 1003, 1040, 1033, 1031), (2047, 1990, 2000, 2048, 2048, 2048)],
         4096: [(2030, 2050, 2040, 2070, 2081, 2077), (4090, 4000, 4090, 4096, 4096, 4096)]}


def compare_to_restatement(v, o, size, res, sizes=None):
    finest = res.bit_length() - 1
    got = voxels.lookup_outputs(lambda p, ms: lookups_engine(v, p, ms), size, finest, seed=3, sizes=sizes)
    want = voxels.lookup_outputs(o.containing_voxels, size, finest, seed=3, sizes=sizes)
    assert_same(got, want)
    for b in CROPS.get(res, []) + mvp.BOXES.get(res, []):
        want = voxels.dense_from_lookups(lambda p: o.containing_voxels(p, -1.0), size, res, b)
        assert_same(dense_engine(v, b), want)


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_shapes_against_the_restatement(name):
    case = SHAPES[name]
    cfg = dict(case[0], **mvp.color_kw(case[4]))
    f = Fused(cfg, mvp.stream(case), pool_log2=19 if cfg["xres"] >= 1024 else 18)
    compare_to_restatement(f.v, f.o, f.size, f.res)


@pytest.mark.parametrize("cid", ["K1", "K4", "K5"])
def test_carved_volumes_read_as_fresh(cid):
    from tests.dynamic_cases import CASES
    case = CASES[cid]
    cfg = case.config()
    f = Fused(cfg, case.frames(), pool_log2={256: 17, 2048: 18, 4096: 19}[case.res])
    compare_to_restatement(f.v, f.o, f.size, f.res)


def test_loaded_volume(tmp_path):
    case = mvp.CASES["pin_256_5_9_rgb"]
    v = engine(dict(case[0], **mvp.color_kw(case[4])))
    mvp.fuse(v_adapter(v), case)
    path = str(tmp_path / "v.vol")
    v.save(path)
    w = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
    w.load(path)
    assert_same(outputs_engine(w, case), outputs_engine(v, case))


# ---- whole volumes, protocol, ordering, refusals --------------------------------------------------------------------------
def test_whole_256_volume_equals_device_lookups():
    case = mvp.CASES["pin_256_5_9_rgb"]
    v = engine(dict(case[0], **mvp.color_kw(case[4])))
    mvp.fuse(v_adapter(v), case)
    res, size = 256, case[0]["xsize"]
    dense = dense_engine(v, (0, 0, 0, res, res, res))
    c = torch.from_numpy(voxels.voxel_centers_1d(size, res, np.arange(res))).cuda()
    pts = torch.stack(torch.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3).contiguous()
    rec = torch.empty(res ** 3 * 44, dtype=torch.uint8, device="cuda")
    v.getContainingVoxelsDevice(pts.data_ptr(), res ** 3, rec.data_ptr())
    v.sync()
    r = rec.cpu().numpy().view(pkg.VOXEL_DTYPE).reshape(res, res, res)
    assert np.array_equal(dense["d"].view(np.uint32), r["d"].view(np.uint32))
    assert np.array_equal(dense["w"].view(np.uint32), r["w"].view(np.uint32))
    assert np.array_equal(dense["rgb"], np.stack([r["r"], r["g"], r["b"]], -1))
    assert np.array_equal(dense["level"], r["level"].astype(np.int8))
    assert (r["level"] > 0).all() and (dense["w"] > 0).sum() > 10000


def test_each_output_alone():
    case = mvp.CASES["pin_2048_2_3_rgb"]
    v = engine(dict(case[0], **mvp.color_kw(case[4])))
    mvp.fuse(v_adapter(v), case)
    box = (1000, 1010, 990, 1043, 1037, 1033)
    full = dense_engine(v, box)
    for k in full:
        assert dense_engine(v, box, outputs=(k,))[k].tobytes() == full[k].tobytes(), k


def test_lookups_queued_after_a_device_batch_see_the_whole_batch():
    case = mvp.CASES["pin_256_5_9_rgb"]
    cfg = dict(case[0], **mvp.color_kw(case[4]))
    ref = engine(cfg)
    mvp.fuse(v_adapter(ref), case)
    v = engine(cfg)
    fr = list(mvp.stream(case))
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fr]
    torch.cuda.synchronize()
    H, W, nf = dev[0].shape
    box = (90, 101, 77, 131, 140, 109)
    pts = voxels.point_sets(3.0, 8)["uniform"]
    x = torch.from_numpy(pts).cuda()
    rec = torch.empty(len(pts) * 44, dtype=torch.uint8, device="cuda")
    d = torch.empty(41 * 39 * 32, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    v.integrateBatchDevice([t.data_ptr() for t in dev], H, W, 4 * nf, [p for p, _ in fr], rgba_off=16)
    v.getContainingVoxelsDevice(x.data_ptr(), len(pts), rec.data_ptr())             # no sync in between
    v.extractDenseDevice(box, d_d=d.data_ptr())
    v.sync()
    assert rec.cpu().numpy().tobytes() == ref.getContainingVoxels(pts).tobytes()
    assert d.cpu().numpy().tobytes() == dense_engine(ref, box, outputs=("d",))["d"].tobytes()


def _raw(v, box=None, outs=(True, True, True, True), lookup=True):
    """the dense crop (and, with lookup, a point lookup) through the C ABI into guarded buffers: (rc, rc, no byte changed)"""
    lib = pkg.load_library()
    n = 64
    bufs = [guarded(n * 4), guarded(n * 4), guarded(n * 3), guarded(n)]
    args = [b.data_ptr() if o else None for b, o in zip(bufs, outs)]
    import ctypes
    b = (ctypes.c_int32 * 6)(*(box or (0, 0, 0, 4, 4, 4)))
    rc = lib.b200tsdf_dense_device(v._h, b, *[None if a is None else ctypes.c_void_p(a) for a in args])
    x = torch.zeros(n * 3, dtype=torch.float32, device="cuda")
    r2 = guarded(44 * n)
    rc2 = None
    if lookup:
        rc2 = lib.b200tsdf_containing_voxels_device(v._h, ctypes.c_void_p(x.data_ptr()), n, ctypes.c_float(-1.0), ctypes.c_void_p(r2.data_ptr()))
    torch.cuda.synchronize()
    untouched = all((t.cpu().numpy() == SENTINEL).all() for t in bufs + [r2])
    return rc, rc2, untouched


def test_refusals_write_nothing():
    cfg = dict(CFG_256, integrate_color=1)
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=16)                                 # before reset()
    for k, x in cfg.items():
        setattr(v._cfg, k, x)
    v._push()
    assert _raw(v) == (ESTATE, ESTATE, True)
    s = pkg.TSDFVolumeOctree(device=0, pool_log2=16, shard_rank=0, shard_count=2)    # a shard
    for k, x in cfg.items():
        setattr(s._cfg, k, x)
    s._push()
    s.reset()
    assert _raw(s) == (ESTATE, ESTATE, True)
    v.reset()
    for box in [(0, 0, 0, 0, 4, 4), (-1, 0, 0, 4, 4, 4), (0, 0, 0, 257, 4, 4), (5, 0, 0, 4, 4, 4), (0, 0, 250, 4, 4, 257)]:
        rc, _, untouched = _raw(v, box, lookup=False)
        assert rc == EINVAL and untouched, box
    rc, _, untouched = _raw(v, outs=(False, False, False, False), lookup=False)
    assert rc == EINVAL and untouched
    assert v.getContainingVoxels(np.zeros((0, 3), np.float32)).size == 0                # n == 0 is a no-op
