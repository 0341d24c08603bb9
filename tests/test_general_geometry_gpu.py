"""The CUDA engine under general inputs (tests/general_cases.py) against the restatement, bit for bit: nodes, addObservation
counts frame by frame, cull masks, renders and meshes in the reference's order.  Every case runs through the route reset()
picks, through the general depth-first kernel (debug_flags bit 0), and for G1 and G3 through integrateBatchDevice in four
equal batches: the engine keeps one captured graph per half of the record ring and batch size, so the first two batches
capture a graph on each half and the last two relaunch them with rewritten records.  The reference build's digests
(tests/golden/general_pins.json) are replayed against the engine directly."""
import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from tests.common import digests
from tests.general_cases import CASES, IDS, OracleAdapter, outputs
from tests.test_general_geometry import PINS, port_digests

pytestmark = pytest.mark.gpu


def pool_log2(case):
    return {256: 17, 512: 18, 2048: 18, 4096: 19}[case.res]


BATCHES = 4


class EngineAdapter:
    """the engine behind the interface of tests/general_cases.py.  general: the general depth-first update kernel only;
    batch: frames are fused by integrateBatchDevice in BATCHES equal batches, inside a profile_begin / profile_end region"""

    def __init__(self, case, general=False, batch=False):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2(case))
        for k, x in case.config().items():
            setattr(v._cfg, k, x)
        v._cfg.debug_flags = 1 if general else 0
        v._push()
        v.reset()
        self.v, self.case = v, case
        self.batch = len(case.poses) * case.repeat // BATCHES if batch else 0
        assert not batch or self.batch * BATCHES == len(case.poses) * case.repeat
        self.pending = []
        if batch:
            v.profile_begin()

    def integrate(self, cloud, pose):
        if not self.batch:
            self.v.integrateCloud(cloud, None, pose)
            return
        import torch
        self.pending.append((torch.from_numpy(np.ascontiguousarray(cloud)).cuda(), pose))
        if len(self.pending) == self.batch:
            dev, poses = zip(*self.pending)
            H, W, nf = dev[0].shape
            torch.cuda.synchronize()
            self.v.integrateBatchDevice([d.data_ptr() for d in dev], H, W, 4 * nf, poses, rgba_off=16 if nf >= 8 else -1)
            self.v.sync()
            self.pending = []

    def n_updates(self):
        return None if self.batch else self.v.stats().n_updates

    def levels(self):
        st = self.v.stats()
        return st.coarse_level, st.finest_level

    def dump_nodes(self):
        assert not self.pending
        return self.v.download_nodes()

    def cull(self, pose):
        return self.v.getFrustumCulledVoxels(pose)

    def render(self, pose, ds, colored):
        return self.v.renderColoredView(pose, ds) if colored else (self.v.renderView(pose, ds), None)

    def mesh(self, wmin, cm):
        mc = pkg.MarchingCubesTSDFOctree()
        mc.setInputTSDF(self.v)
        mc.setMinWeight(wmin)
        mc.setColorByRGB(cm == 1)
        v, rgb, _ = mc.reconstruct()
        return v, rgb


def differing(got, want):
    return [k for k in want if got.get(k) != want[k]] + [k for k in got if k not in want]


ROUTES = [(cid, "reset") for cid in IDS] + [(cid, "general") for cid in IDS] + [("G1", "batch"), ("G3", "batch")]


@pytest.mark.parametrize("cid,route", ROUTES)
def test_engine_matches_restatement(cid, route):
    case = CASES[cid]
    e = EngineAdapter(case, general=route == "general", batch=route == "batch")
    got = digests(outputs(case, e))
    want = port_digests(cid)
    if route == "batch":                       # one count per batch: the last frame's
        want = {k: v for k, v in want.items() if k != "n_updates"}
        assert e.n_updates() is None and e.v.stats().n_updates == outputs_last_count(cid)
        # one graph launch per batch: two captures (one per ring half), each launched twice
        assert e.v.profile_end().graph_launches == BATCHES
    assert differing(got, want) == []
    # the reference build's own digests, replayed against the engine
    assert differing({k: v for k, v in got.items() if k != "n_updates"}, PINS[cid]) == []


_counts = {}


def outputs_last_count(cid):
    if cid not in _counts:
        a = OracleAdapter(CASES[cid])
        for pose, cloud in CASES[cid].frames():
            a.integrate(cloud, pose)
        _counts[cid] = a.n_updates()
    return _counts[cid]


def launches_per_frame(case, **cfg):
    """total kernel launches per integrate call for `case` with the configuration fields in `cfg` overridden"""
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2(case))
    for k, x in {**case.config(), **cfg}.items():
        setattr(v._cfg, k, x)
    v._push()
    v.reset()
    pose, cloud = next(case.frames())
    v.profile_begin()
    for _ in range(2):
        v.integrateCloud(cloud, None, pose)
    prof = v.profile_end()
    assert prof.n_frames == 2
    return prof.total_launches / prof.n_frames


def test_division_outside_its_exact_range_takes_the_general_kernel():
    """D1 (max_dist_neg = 1.2e-38) is outside Params::exact_div_ok: reset() must route it to the general depth-first kernel,
    which divides with the IEEE division, not to the brick kernels.  The same grid with an in-range truncation limit takes the
    brick kernels, also with the integrate program's default sensor bounds (min_sensor_dist = 0): those are not operands of
    the division."""
    case = CASES["D1"]
    general = launches_per_frame(case, debug_flags=1)
    assert launches_per_frame(case) == general
    brick = launches_per_frame(case, max_dist_neg=0.03)
    assert brick > general
    assert launches_per_frame(case, max_dist_neg=0.03, min_sensor_dist=0.0) == brick
