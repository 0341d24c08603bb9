"""Frames that overlap on the device: on the route whose supercells are the culled coarse cells, a frame's k_front pre-splits a
pixel as soon as the previous frame has folded that pixel's supercell, not after the previous frame's whole k_celltop_up
(FoldState, brick_kernels.cuh).  The next frame's k_front then writes its pixel plane, cell queue and counter set while the
previous frame still runs, so these tests drive each of those buffers and the gate itself through graph-replayed batches, in
which consecutive frames are chained by programmatic dependent launch.

* Plane hazard: two poses whose views share almost no pixels, alternating, so every plane entry changes from frame to frame.
* Per-frame statistics on the bench stream (2048^3 / 10 m, colour), through two 32-frame batches and then one frame per call.
* Dynamic scenes K1, K4 and K6 (prunes and re-splits in k_celltop_up) in single batches, against the reference's pins.
* Which k_front runs, read from the debug counters of b200tsdf_debug_timing.
* reset () and load () between batches."""
import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, assert_same_nodes, digests
from tests.dynamic_cases import CASES, node_digest_bytes, outputs
from tests.test_dynamic_scenes import PINS
from tests.test_dynamic_scenes_gpu import EngineAdapter, debug_timing, differing

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def engine(cfg, pool_log2=17, color=True, flags=0):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
    v.setCameraIntrinsics(525.0, 525.0, cfg["cx"], cfg["cy"])
    v.setIntegrateColor(color)
    v._cfg.debug_flags = flags
    v._push()
    v.reset()
    return v


def oracle(cfg, color=True):
    o = OracleVolume(**cfg, integrate_color=int(color))
    o.reset()
    return o


def batch(v, clouds, poses):
    """one integrateBatchDevice call: one graph launch for all the frames"""
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in clouds]
    torch.cuda.synchronize()
    H, W, nf = clouds[0].shape
    v.integrateBatchDevice([d.data_ptr() for d in dev], H, W, 4 * nf, poses, rgba_off=16 if nf >= 8 else -1)
    v.sync()


def same_stats(v, o):
    a, b = v.stats(), o.stats()
    assert (a.n_updates, a.n_culled_cells) == (b.n_add_observation, b.n_culled_cells)


def stream(scene, idx, total=100, seed=7):
    poses = [synth.orbit_pose(scene, f, total) for f in idx]
    return poses, [synth.make_frame(scene, p, CAM, color=True, noise_seed=seed, frame=i) for i, p in enumerate(poses)]


def test_alternating_views_plane_hazard():
    """Opposite sides of the orbit, alternating: consecutive frames see different walls, so every plane entry changes.  Two
    handles take the same 12 frames in calls of 2 frames, offset by one, so that every frame is the overlapped second frame of a
    call on one of them: the statistics after every call, and every node, must equal the restatement's."""
    poses, clouds = stream(synth.S1, [0, 50] * 6)
    orc = oracle(CFG_512)
    want_stats, want_nodes = [], []
    for p, c in zip(poses, clouds):
        orc.integrate(c, p)
        s = orc.stats()
        want_stats.append((s.n_add_observation, s.n_culled_cells))
        want_nodes.append(orc.dump_nodes())
    for first in (2, 1):
        v = engine(CFG_512)
        cuts = [0] + list(range(first, len(poses) + 1, 2))
        if cuts[-1] != len(poses):
            cuts.append(len(poses))
        for a, b in zip(cuts, cuts[1:]):
            batch(v, clouds[a:b], poses[a:b])
            st = v.stats()
            assert (st.n_updates, st.n_culled_cells) == want_stats[b - 1], (first, b)
            assert_same_nodes(want_nodes[b - 1], v.download_nodes(), rgb=True)


def test_bench_stream_statistics_per_call():
    """The first 64 frames of the bench stream as two 32-frame graph launches, then 8 frames one per call: stats () after every
    call equals the restatement's counts for that call's last frame, and the nodes are bit-identical at the end."""
    poses = [synth.orbit_pose(synth.S2, f, 100) for f in range(72)]
    clouds = [synth.make_frame(synth.S2, p, CAM, color=True, noise_seed=12345, frame=f) for f, p in enumerate(poses)]
    v, orc = engine(CFG_2048, 18), oracle(CFG_2048)
    for k0 in (0, 32):
        for f in range(k0, k0 + 32):
            orc.integrate(clouds[f], poses[f])
        batch(v, clouds[k0:k0 + 32], poses[k0:k0 + 32])
        same_stats(v, orc)
    for f in range(64, 72):
        orc.integrate(clouds[f], poses[f])
        v.integrateCloud(clouds[f], None, poses[f])
        same_stats(v, orc)
    assert_same_nodes(orc.dump_nodes(), v.download_nodes(), rgb=True)


class OneCall(EngineAdapter):
    """the engine behind the interface of tests/dynamic_cases.py, every frame held back until the state is read, then fused
    by one integrateBatchDevice call"""

    def __init__(self, case):
        super().__init__(case)
        self.frames = []

    def integrate(self, cloud, pose):
        self.frames.append((cloud, pose))

    def flush(self):
        if self.frames:
            clouds, poses = zip(*self.frames)
            batch(self.v, list(clouds), list(poses))
            self.frames = []

    def n_updates(self):
        return None

    def dump_nodes(self):
        self.flush()
        return self.v.download_nodes()

    def render(self, pose, ds, colored):
        self.flush()
        return super().render(pose, ds, colored)

    def mesh(self, wmin, cm):
        self.flush()
        return super().mesh(wmin, cm)


@pytest.mark.parametrize("cid", ["K1", "K4"])
def test_dynamic_scenes_in_one_batch(cid):
    case = CASES[cid]
    got = digests(outputs(case, OneCall(case)))
    assert differing(got, {k: x for k, x in PINS[cid].items() if k != "n_updates"}) == []


def test_dynamic_scene_k6_every_prefix_in_one_batch():
    """K6 pins the nodes after every one of its 9 frames, all at one pose (every pixel waits for its cell's fold): the prefix
    of each length, fused by one call on a fresh handle, matches the pin of its last frame"""
    case = CASES["K6"]
    frames = list(case.frames())
    for n in range(1, len(frames) + 1):
        e = OneCall(case)
        for pose, cloud in frames[:n]:
            e.integrate(cloud, pose)
        got = digests({"x": node_digest_bytes(e.dump_nodes())})["x"]
        assert got == PINS["K6"][f"frame{n - 1}_nodes"], n


def routes(v, clouds, poses):
    """(frames whose k_front waited per supercell, frames whose k_front waited for the previous frame) over one batch"""
    batch(v, clouds, poses)
    d = debug_timing(v)
    return int(d[11]), int(d[12])


def test_route_selection():
    poses, clouds = stream(synth.S1, range(0, 8, 2))
    v = engine(CFG_512)
    debug_timing(v)                                         # arm the counters
    assert routes(v, clouds, poses) == (3, 1)               # the first frame after reset () has no published marks to wait on
    assert routes(v, clouds, poses) == (4, 0)
    # out-of-domain writes move the handle to the general kernel, whose k_front waits
    v.setContainingVoxelsData(np.zeros((1, 3), np.float32), 1e30, 1.0)
    assert routes(v, clouds, poses) == (0, 4)
    v.reset()
    assert routes(v, clouds, poses) == (3, 1)
    # debug_flags bit 0 (general kernel), C < SL (1024^3 / 3 m: an upper level above the supercells), C > SL (256^3 / 3 m)
    for cfg, flags in ((CFG_512, 1), (dict(CFG_512, xres=1024, yres=1024, zres=1024), 0), (CFG_256, 0)):
        w = engine(cfg, 19, flags=flags)
        debug_timing(w)
        assert routes(w, clouds, poses) == (0, 4), (cfg["xres"], flags)


def test_reset_and_load_mid_stream(tmp_path):
    """reset () between batches, and load () of a volume saved earlier, continue the stream bit for bit"""
    poses, clouds = stream(synth.S1, range(0, 48, 4))
    orc = oracle(CFG_512)
    for p, c in zip(poses[:4], clouds[:4]):
        orc.integrate(c, p)
    path = str(tmp_path / "mid.vol")
    orc.save(path)
    for p, c in zip(poses[4:8], clouds[4:8]):
        orc.integrate(c, p)
    after8 = orc.dump_nodes()
    v = engine(CFG_512)
    batch(v, clouds[8:], poses[8:])
    v.load(path)
    batch(v, clouds[4:8], poses[4:8])
    same_stats(v, orc)
    assert_same_nodes(after8, v.download_nodes(), rgb=True)
    fresh = oracle(CFG_512)
    for p, c in zip(poses[6:], clouds[6:]):
        fresh.integrate(c, p)
    v.reset()
    batch(v, clouds[6:], poses[6:])
    same_stats(v, fresh)
    assert_same_nodes(fresh.dump_nodes(), v.download_nodes(), rgb=True)
