"""getFxn / getGradient / getHessian (k_query) and getTSDFValue (k_interpolate) of the CUDA engine against the digests of the
reference's own methods (tests/golden/query_pins.json, tools/make_query_pins.py), bit for bit, on the volumes and point
sets of tests/query_cases.py: exact centre and face ties, their ulp neighbours, the border layers of the grid, neighbourhoods
of mixed leaf depth, NaN, infinities and coordinates beyond 2^31 voxels, on every tier shape.

Every call goes through the host entry point (b200tsdf_query, b200tsdf_interpolate) and the device entry point
(b200tsdf_query_device, b200tsdf_interpolate_device, into buffers with guard bytes), which must agree byte for byte; the
outputs of a point that is not ok, and outputs that were not asked for, must keep the caller's sentinel.  Only tests/golden/
is read; when a digest differs the restatement names the first differing point."""
import ctypes
import json
import os

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from tests import query_cases as qc
from tests.common import digests

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "query_pins.json")))["cases"]
SENTINEL = np.float32(-1234.5)                  # what every output buffer holds before a call
GUARD = 1024                                    # floats (or bytes of `ok`) of sentinel after every device output's extent
OK_SENTINEL = 0xA5


def engine(volume, flags=0, **kw):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=volume.pool_log2, **kw)
    for k, x in volume.config.items():
        setattr(v._cfg, k, x)
    v._cfg.debug_flags = flags
    v._push()
    v.reset()
    return v


def fuse(v, volume, route="cloud"):
    """route "cloud": integrateCloud frame by frame; "batch": every frame in one integrateBatchDevice call"""
    fr = list(volume.frames())
    if route == "cloud":
        for pose, cloud in fr:
            v.integrateCloud(cloud, None, pose)
    else:
        dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fr]
        torch.cuda.synchronize()
        H, W, nf = dev[0].shape
        v.integrateBatchDevice([d.data_ptr() for d in dev], H, W, 4 * nf, [p for p, _ in fr], rgba_off=16 if nf >= 8 else -1)
        v.sync()
    return v


def _dev(shape):
    n = int(np.prod(shape))
    return torch.full((n + GUARD,), float(SENTINEL), dtype=torch.float32, device="cuda")


def _back(t, shape):
    n = int(np.prod(shape))
    h = t.cpu().numpy()
    assert (h[n:] == SENTINEL).all(), "a float past the extent changed"
    return h[:n].reshape(shape)


class EngineAdapter:
    """a fused engine handle behind the interface of tests/query_cases.py; every call checks host against device entry point
    and the sentinels"""

    def __init__(self, v):
        self.v, self.lib = v, v._lib

    def dump_nodes(self):
        return self.v.download_nodes()

    def query_device(self, pts, what, mode):
        n = len(pts)
        shapes = ((n,), (n, 3), (n, 3, 3))
        x = torch.from_numpy(np.ascontiguousarray(pts)).cuda() if n else torch.zeros(3, device="cuda")
        bufs = [_dev(s) for s in shapes]
        ok = torch.full((n + GUARD,), OK_SENTINEL, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        self.v.queryDevice(x.data_ptr(), n, ok.data_ptr(), what, mode, *[b.data_ptr() if what & (1 << k) else None for k, b in enumerate(bufs)])
        self.v.sync()
        okh = ok.cpu().numpy()
        assert (okh[n:] == OK_SENTINEL).all() and np.isin(okh[:n], (0, 1)).all()
        return [_back(b, s) for b, s in zip(bufs, shapes)] + [okh[:n].astype(bool)]

    def query_host(self, pts, what, mode):
        pts = np.ascontiguousarray(pts, np.float32)
        n = len(pts)
        val, grad, hess = (np.full(s, SENTINEL, np.float32) for s in ((n,), (n, 3), (n, 3, 3)))
        ok = np.full(n, OK_SENTINEL, np.uint8)
        p = lambda a, on=True: a.ctypes.data_as(ctypes.c_void_p) if on else None
        self.v._check(self.lib.b200tsdf_query(self.v._h, p(pts), n, what, mode, p(val, what & 1), p(grad, what & 2), p(hess, what & 4), p(ok)))
        assert np.isin(ok, (0, 1)).all()
        return [val, grad, hess, ok.astype(bool)]

    def query(self, pts, what, mode):
        host, dev = self.query_host(pts, what, mode), self.query_device(pts, what, mode)
        for k, (h, d) in enumerate(zip(host, dev)):
            assert h.tobytes() == d.tobytes(), ("host and device entry points differ", what, mode, k)
        ok = host[3]
        for k in range(3):
            if what & (1 << k):
                assert (host[k][~ok] == SENTINEL).all(), ("an output of a point that is not ok was written", what, mode, k)
            else:
                assert (host[k] == SENTINEL).all(), ("an output that was not asked for was written", what, mode, k)
        return host

    def interpolate_device(self, pts, valid):
        n = len(pts)
        x = torch.from_numpy(np.ascontiguousarray(pts)).cuda() if n else torch.zeros(3, device="cuda")
        val = _dev((n,))
        ok = torch.full((n + GUARD,), OK_SENTINEL, dtype=torch.uint8, device="cuda")
        ok[:n] = torch.from_numpy(np.ascontiguousarray(valid, np.uint8)).cuda()
        torch.cuda.synchronize()
        self.v.getTSDFValueDevice(x.data_ptr(), n, val.data_ptr(), ok.data_ptr())
        self.v.sync()
        okh = ok.cpu().numpy()
        assert (okh[n:] == OK_SENTINEL).all()
        return _back(val, (n,)), okh[:n].astype(bool)

    def interpolate(self, pts, valid):
        pts = np.ascontiguousarray(pts, np.float32)
        n = len(pts)
        val, ok = np.full(n, SENTINEL, np.float32), np.ascontiguousarray(valid, np.uint8).copy()
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        self.v._check(self.lib.b200tsdf_interpolate(self.v._h, p(pts), n, p(val), p(ok)))
        dval, dok = self.interpolate_device(pts, valid)
        assert val.tobytes() == dval.tobytes() and np.array_equal(ok.astype(bool), dok), "host and device entry points differ"
        assert not (ok.astype(bool) & ~np.asarray(valid, bool)).any()      # the flag is only ever cleared
        return val, ok.astype(bool)


def explain(e, volume, sets, keys):
    """for each differing digest: the first point at which the engine and the restatement differ, its voxel index, both results"""
    o = qc.OracleAdapter(volume, "port")
    lines = []
    for key in keys:
        name, _, call = key.partition(".")
        if name not in sets or not (call.startswith("query_w") or call.startswith("tsdf_")) or call.count("."):
            lines.append(f"{key}: differs")
            continue
        pts = sets[name]
        if call.startswith("query_w"):
            what, mode = int(call[7]), int(call[-1])
            got, want = e.query_host(pts, what, mode), o.query(pts, what, mode)
            cols = [g.reshape(len(pts), -1) for g in got[:3]], [w.reshape(len(pts), -1) for w in want[:3]]
            bad = got[3] != want[3]
            for k in range(3):
                if what & (1 << k):
                    bad |= got[3] & want[3] & (cols[0][k].view(np.uint32) != cols[1][k].view(np.uint32)).any(1)
            show = lambda r, i: (bool(r[3][i]), [a[i].tolist() for a in r[:3]])
        else:
            vin = qc.valid_in(call[5:], len(pts))
            got, want = e.interpolate(pts, vin), o.interpolate(pts, vin)
            bad = (got[1] != want[1]) | (np.isnan(got[0]) != np.isnan(want[0])) | (~np.isnan(got[0]) & (got[0].view(np.uint32) != want[0].view(np.uint32)))
            show = lambda r, i: (bool(r[1][i]), float(r[0][i]))
        if not bad.any():
            lines.append(f"{key}: the engine equals the restatement, the pin differs from both")
            continue
        i = int(np.argmax(bad))
        vox = np.floor(qc.index_expr(volume.size, volume.res, pts[i])).tolist()
        lines.append(f"{key}: {int(bad.sum())} points differ; first #{i} {pts[i].tolist()} (hex {pts[i].view(np.uint32).tolist()}) "
                     f"voxel {vox}: engine {show(got, i)} restatement {show(want, i)}")
    return "\n".join(lines)


def assert_pinned(v, volume):
    e = EngineAdapter(v)
    nodes = e.dump_nodes()
    sets = qc.point_sets(volume, nodes)
    got = digests(qc.outputs(e, volume, sets, qc.LeafIndex(nodes, volume.res)))
    bad = [k for k in PINS[volume.id] if got.get(k) != PINS[volume.id][k]] + [k for k in got if k not in PINS[volume.id]]
    assert not bad, "\n" + explain(e, volume, sets, bad[:12])
    return e, sets


@pytest.mark.parametrize("vid", qc.IDS)
def test_engine_reproduces_reference_queries(vid):
    volume = qc.VOLUMES[vid]
    assert_pinned(fuse(engine(volume), volume), volume)


@pytest.mark.parametrize("vid", ["Q256", "Q2048"])
def test_any_number_of_points(vid):
    """n = 0, 1, one under, at and over the block size, and a million and three (the grid's tail): every point's results are
    those of the same point in the pinned run, and nothing past the extent is written"""
    volume = qc.VOLUMES[vid]
    e, sets = assert_pinned(fuse(engine(volume), volume), volume)
    base = np.concatenate([sets[k] for k in ("special", "border", "centres", "faces", "mixed", "random")])
    want = e.query_host(base, 7, 1)
    vin = qc.valid_in("mix", len(base))
    want_t = e.interpolate(base, vin)
    assert 0 < want[3].sum() < len(base)
    for n in (1, 127, 128, 129, 1_000_003):
        idx = np.arange(n) % len(base)
        got = e.query(base[idx], 7, 1)
        for g, w in zip(got, want):
            assert g.tobytes() == w[idx].tobytes(), n
        val, ok = e.interpolate(base[idx], vin[idx])
        assert val.tobytes() == want_t[0][idx].tobytes() and np.array_equal(ok, want_t[1][idx]), n
    none = np.zeros((0, 3), np.float32)
    for what in qc.WHATS:
        assert e.query(none, what, 0)[3].size == 0                      # host and device: accepted, nothing written
    assert e.interpolate(none, np.zeros(0, np.uint8))[0].size == 0


@pytest.mark.parametrize("vid", ["Q256", "Q2048"])
def test_saved_and_loaded_volume(vid, tmp_path):
    volume = qc.VOLUMES[vid]
    v = fuse(engine(volume), volume)
    path = str(tmp_path / "v.vol")
    v.save(path)
    w = pkg.TSDFVolumeOctree(device=0, pool_log2=volume.pool_log2)
    w.load(path)
    assert_pinned(w, volume)


def test_three_shards_gathered_into_one_handle():
    """Q2048's coarse cells are the root arrays, so its shards can be exported and imported"""
    volume = qc.VOLUMES["Q2048"]
    full = engine(volume)
    for rank in range(3):
        s = fuse(engine(volume, shard_rank=rank, shard_count=3), volume)
        full.import_shard(s.export_shard())
    assert_pinned(full, volume)


@pytest.mark.parametrize("route,flags", [("batch", 0), ("cloud", 1), ("batch", 1)])
def test_every_write_route_reads_the_same(route, flags):
    """Q2048 fused by integrateBatchDevice, and by the general depth-first kernel (debug_flags bit 0), reads as the volume
    fused by integrateCloud does (test_engine_reproduces_reference_queries): the read pins hold for every write route"""
    volume = qc.VOLUMES["Q2048"]
    assert_pinned(fuse(engine(volume, flags), volume, route), volume)
