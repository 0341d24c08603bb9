"""The CUDA engine on scenes that change while they are fused (tests/dynamic_cases.py), where pre-existing children are
pruned and nodes re-split in the same call.

* Parity: every case, bit for bit against the restatement and against the reference build's digests
  (tests/golden/dynamic_pins.json), through the route reset() picks, the general depth-first kernel (debug_flags bit 0),
  the per-level upper sweeps (bit 1), and for K1 to K5 integrateBatchDevice in graph-replayed batches (K1, K4 and K5
  also with the general kernel).  The per-frame routes compare addObservation counts frame by frame.
* Coverage on the device: the diagnostic counters of k_celltop_up show that the slow paths these streams exist for ran.
* The fresh invariant on raw storage: after every frame of the carve phase, every node that does not exist, in every
  claimed brick, is exactly in the constructor state.
* Pool pressure: K1 and K4 with the hash table loaded to between 0.5 and 0.85 give the same nodes as with a large pool."""
import ctypes as C
import math

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from tests.common import digests
from tests.dynamic_cases import CASES, IDS, OracleAdapter, outputs
from tests.test_dynamic_scenes import PINS, port_digests

pytestmark = pytest.mark.gpu


def pool_log2(case):
    return {256: 17, 512: 18, 2048: 18, 4096: 19}[case.res]


BATCH = 2                                          # frames per integrateBatchDevice call (every batched case has an even number)


class EngineAdapter:
    """the engine behind the interface of tests/dynamic_cases.py.  flags: b200tsdf_config.debug_flags; batch: frames are
    fused by integrateBatchDevice, BATCH at a time, inside a profile_begin / profile_end region"""

    def __init__(self, case, flags=0, batch=False, pool=None):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool or pool_log2(case), track_variance=case.track_variance)
        for k, x in case.config().items():
            setattr(v._cfg, k, x)
        v._cfg.debug_flags = flags
        v._push()
        v.reset()
        self.v, self.case, self.batch = v, case, batch
        self.pending = []
        if batch:
            v.profile_begin()

    def integrate(self, cloud, pose):
        if not self.batch:
            self.v.integrateCloud(cloud, None, pose)
            return
        import torch
        self.pending.append((torch.from_numpy(np.ascontiguousarray(cloud)).cuda(), pose))
        if len(self.pending) == BATCH:
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


FLAGS = {"reset": 0, "general": 1, "upper": 2}
BATCHED = {"batch": 0, "general_batch": 1}         # integrateBatchDevice on the route reset() picks / the general kernel
# K2 (variance) and K3 (RGBNormalized) take the general kernel, and general_batch forces it on brick-route shapes: their
# batches are graph launches as well.  K6 pins its nodes after every one of its 9 frames, so it is not fused in pairs.
ROUTES = [(cid, r) for r in FLAGS for cid in IDS] + [(cid, "batch") for cid in ("K1", "K2", "K3", "K4", "K5")] \
    + [(cid, "general_batch") for cid in ("K1", "K4", "K5")]


@pytest.mark.parametrize("cid,route", ROUTES)
def test_engine_matches_restatement(cid, route):
    case = CASES[cid]
    e = EngineAdapter(case, flags={**FLAGS, **BATCHED}[route], batch=route in BATCHED)
    got = digests(outputs(case, e))
    want = port_digests(cid)
    if route in BATCHED:                       # one count per batch: the last frame's
        want = {k: v for k, v in want.items() if k != "n_updates"}
        assert e.v.profile_end().graph_launches == len(case.poses) // BATCH
    assert differing(got, want) == []
    assert differing({k: v for k, v in got.items() if k != "n_updates"}, PINS[cid]) == []


# ---- coverage on the device ------------------------------------------------------------------------------------------
def debug_timing(v):
    """b200tsdf_debug_timing: the first call arms k_celltop_up's diagnostic counters on this handle (and drops its captured
    graphs); every call returns and clears them.  [6..10]: slow level-2 nodes, slow level-1 nodes, cell leaf visits, cell
    fall-throughs, cells folded."""
    lib = v._lib
    lib.b200tsdf_debug_timing.argtypes = [C.c_void_p, C.c_void_p]
    out = np.zeros(16, np.uint64)
    v._check(lib.b200tsdf_debug_timing(v._h, out.ctypes.data_as(C.c_void_p)))
    return out


_coverage = {}


def coverage(cid):
    """per stream, on a handle of its own: the sums of debug counters [6..10], of stats.reserved, n_slow_visits and n_bail
    (the last three are always 0)"""
    if cid not in _coverage:
        case = CASES[cid]
        e = EngineAdapter(case)
        debug_timing(e.v)
        dbg = np.zeros(5, np.int64)
        folds = slow = bail = 0
        for pose, cloud in case.frames():
            e.integrate(cloud, pose)
            st = e.v.stats()
            folds += st.reserved
            slow += st.n_slow_visits
            bail += st.n_bail
            dbg += debug_timing(e.v)[6:11].astype(np.int64)
        _coverage[cid] = dict(slow2=int(dbg[0]), slow1=int(dbg[1]), cell_leaf=int(dbg[2]), fall_through=int(dbg[3]),
                              folded=int(dbg[4]), upper_folds=folds, slow_visits=slow, bail=bail)
    return _coverage[cid]


def test_device_reaches_the_slow_paths():
    """Each of k_celltop_up's slow paths runs on some case: slow level-2 and level-1 nodes (pre-existing children pruned
    above the brick's finest level), leaf visits of a cell, and fall-through updates of a cell whose children were pruned.
    K2 and K3 take the general kernel (variance state, RGBNormalized payload), which does not count these."""
    cov = {cid: coverage(cid) for cid in IDS}
    print({cid: c for cid, c in cov.items()})
    for k in ("slow2", "slow1", "cell_leaf", "fall_through"):
        assert any(c[k] > 0 for c in cov.values()), (k, cov)
    assert any(c["folded"] > 0 for c in cov.values())


def coarse_prunes(vol, case):
    """per frame, the number of coarse-level (level C) nodes whose split flag went from 1 to 0"""
    prev, out = None, []
    for pose, cloud in case.frames():
        vol.integrate(cloud, pose)
        d = vol.dump_nodes()
        sp = d["split"][d["keys"][:, 0] == vol.levels()[0]].astype(bool)
        if prev is not None:
            out.append(int((prev & ~sp).sum()))
        prev = sp
    return out


def test_upper_sweeps_fold_a_carved_region():
    """K5 (4096^3 / 10 m) has a coarse level above the supercells, which only k_upper_down / k_upper_up sweep on the route
    reset() picks.  Coarse nodes whose children were all pruned must lose their split flag in the same frames as in the
    restatement, and some must.  (stats.reserved and n_slow_visits cannot show this: they are always 0.)"""
    case = CASES["K5"]
    dev = coarse_prunes(EngineAdapter(case), case)
    ref = coarse_prunes(OracleAdapter(case), case)
    print("K5 coarse prunes per frame", dev)
    assert dev == ref and sum(dev) > 0
    c = coverage("K5")
    assert c["upper_folds"] == 0 and c["slow_visits"] == 0, c


def test_bail_counter_is_never_written():
    """stats.n_bail is always 0 (no kernel hands block roots to a bail-out list: the prune-then-resplit case is visited in
    place), on every stream.  If it is ever given a meaning again, this test fails and should become a real assertion."""
    for cid in IDS:
        assert coverage(cid)["bail"] == 0


# ---- the fresh invariant on raw storage --------------------------------------------------------------------------------
HEADER = np.dtype([("magic", "<u4"), ("version", "<u4"), ("L", "<i4"), ("C", "<i4"), ("T", "<i4"), ("Rtop", "<i4"),
                   ("color", "<i4"), ("var", "<i4"), ("n_roots", "<u4"), ("n_bricks", "<u4"), ("size", "<f4"), ("pad", "<u4")])
ROOT_REC = np.dtype([("r", "<i4"), ("dw", "<u4", 2), ("split", "u1"), ("rgb", "<u4"), ("M", "<u4"), ("ns", "<i4")])
BN, SW = 584, 20                                    # nodes and split words per brick (tsdf_core.cuh)
FRESH_DW = np.array([-1.0, 0.0], np.float32).view(np.uint32)


def decode_shard(buf):
    """b200tsdf_export_shard's buffer (engine.cu, SHARD_MAGIC): header, root records, then per claimed brick its key,
    {d,w} x 584, 20 split words, colour x 584 (if colour), M x 584 and nsample x 584 (if variance)"""
    hd = np.frombuffer(buf, HEADER, 1)[0]
    assert hd["magic"] == 0x42325348 and hd["version"] == 1
    o = HEADER.itemsize
    roots = np.frombuffer(buf, ROOT_REC, int(hd["n_roots"]), o)
    o += roots.nbytes
    fields = [("key", "<u8"), ("dw", "<u4", (BN, 2)), ("split", "<u4", SW)]
    if hd["color"]:
        fields.append(("rgb", "<u4", BN))
    if hd["var"]:
        fields += [("M", "<u4", BN), ("ns", "<i4", BN)]
    bricks = np.frombuffer(buf, np.dtype(fields), int(hd["n_bricks"]), o)
    assert o + bricks.nbytes == len(buf)
    return hd, roots, bricks


def path_index3(x, y, z):
    j = 0
    for i in (2, 1, 0):
        j = (j << 3) | (((x >> i) & 1) << 2) | (((y >> i) & 1) << 1) | ((z >> i) & 1)
    return j


def bits(words, n):
    return ((words[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(len(words), -1)[:, :n].astype(bool)


def check_fresh_invariant(buf):
    """Work out which nodes exist from the split bits (the root arrays, the parent brick for a brick's root, then each
    brick's level-1 and level-2 words) and assert that every node that does not exist, in every claimed brick, is exactly
    fresh: {d,w} = {-1, 0}, split bit 0, colour 0, M = 0, nsample = 0.  Returns (claimed bricks, existing brick nodes,
    bricks whose root does not exist now)."""
    hd, roots, bricks = decode_shard(buf)
    L, T, Rtop = int(hd["L"]), int(hd["T"]), int(hd["Rtop"])
    assert Rtop == hd["C"] and len(roots) == 8 ** Rtop
    root_split = np.zeros(8 ** Rtop, bool)
    root_split[roots["r"]] = roots["split"] != 0
    keys = bricks["key"].astype(np.uint64)
    tier = (keys >> np.uint64(60)).astype(np.int64) - 1
    bc = np.stack([(keys >> np.uint64(s)) & np.uint64(0xFFFFF) for s in (40, 20, 0)], 1).astype(np.int64)
    assert ((tier >= 0) & (tier < T)).all()
    for t in range(T):                              # the key decodes to a node inside the grid at the brick's root level
        assert (bc[tier == t] < (1 << (L - 3 * (t + 1)))).all()
    index = {int(k): i for i, k in enumerate(keys)}
    split = bricks["split"]
    s1, s2, s3 = bits(split[:, 0:1], 8), bits(split[:, 1:3], 64), bits(split[:, 4:20], 512)
    ex = np.zeros((len(bricks), BN), bool)
    root_exists = np.zeros(len(bricks), bool)
    for t in range(T - 1, -1, -1):                  # parents (higher tiers) first
        for i in np.nonzero(tier == t)[0]:
            x, y, z = (int(v) for v in bc[i])
            if t == T - 1:
                r = (x * (1 << Rtop) + y) * (1 << Rtop) + z
                exists, rsplit = True, root_split[r]
            else:
                pk = ((t + 2) << 60) | ((x >> 3) << 40) | ((y >> 3) << 20) | (z >> 3)
                assert pk in index, f"brick {int(keys[i]):#x} has no claimed parent brick"
                pi, j = index[pk], path_index3(x & 7, y & 7, z & 7)
                exists, rsplit = ex[pi, 72 + j], s3[pi, j]
            root_exists[i] = exists
            ex[i, 0:8] = exists and rsplit
            ex[i, 8:72] = np.repeat(ex[i, 0:8] & s1[i], 8)
            ex[i, 72:] = np.repeat(ex[i, 8:72] & s2[i], 8)
    dead = ~ex
    bad = dead & ~((bricks["dw"][:, :, 0] == FRESH_DW[0]) & (bricks["dw"][:, :, 1] == FRESH_DW[1]))
    assert not bad.any(), f"{bad.sum()} non-existent nodes with stale {{d,w}}"
    if hd["color"]:
        assert not (dead & (bricks["rgb"] != 0)).any(), "non-existent nodes with stale colour"
    if hd["var"]:
        assert not (dead & ((bricks["M"] != 0) | (bricks["ns"] != 0))).any(), "non-existent nodes with stale M / nsample"
    assert not (dead[:, 0:8] & s1).any() and not (dead[:, 8:72] & s2).any(), "split bits of non-existent nodes"
    assert not (dead[:, 72:] & s3).any() and (split[:, 3] == 0).all() and (split[:, 0] >> 8 == 0).all()
    assert not s3[tier == 0].any(), "finest-level nodes carry no split bits"
    return len(bricks), int(ex.sum()), int((~root_exists).sum())


@pytest.mark.parametrize("cid,carve_from", [("K2", 3), ("K4", 1)])
def test_non_existent_nodes_are_fresh_in_raw_storage(cid, carve_from):
    """K2 (512^3 / 3 m, variance state) and K4 (2048^3 / 10 m, colour): grids whose coarse cells are the root arrays, so
    b200tsdf_export_shard works on an unsharded handle.  The decoded existence must also account for every node that
    download_nodes returns."""
    case = CASES[cid]
    e = EngineAdapter(case)
    for f, (pose, cloud) in enumerate(case.frames()):
        e.integrate(cloud, pose)
        if f < carve_from:
            continue
        n_bricks, n_exist, n_orphan = check_fresh_invariant(e.v.export_shard().tobytes())
        nodes = e.v.download_nodes()
        n_root = 8 ** e.v.stats().coarse_level
        assert n_exist + n_root == len(nodes["keys"]), (f, n_exist, n_root, len(nodes["keys"]))
        assert n_bricks == e.v.stats().n_bricks
    print(cid, "claimed bricks", n_bricks, "of which rooted at a node that no longer exists", n_orphan)


# ---- pool pressure -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", ["K1", "K4"])
def test_loaded_pool_gives_the_same_nodes(cid):
    """The other tests size their pools well above what their streams claim, so long linear-probe chains, wrap-around at
    the end of the pool and CAS races between different keys do not occur there.  Here the pool is the smallest power of
    two whose load n_bricks / capacity stays at or below 0.85, which must be at least 0.5.  (K6 claims 1996 bricks on an
    H100, load 0.49 or 0.97 with a power-of-two pool, so the 2048^3 stream K4 runs instead: 10753 bricks, load 0.66.)"""
    case = CASES[cid]
    big = EngineAdapter(case)
    for pose, cloud in case.frames():
        big.integrate(cloud, pose)
    nb = big.v.stats().n_bricks
    k = max(8, math.ceil(math.log2(nb / 0.85)))
    small = EngineAdapter(case, pool=k)
    for pose, cloud in case.frames():
        small.integrate(cloud, pose)
    st = small.v.stats()
    load = st.n_bricks / st.pool_capacity
    print(cid, "bricks", st.n_bricks, "pool_log2", k, "load", round(load, 3))
    assert st.n_bricks == nb and 0.5 <= load <= 0.85, (nb, k, load)
    a, b = big.v.download_nodes(), small.v.download_nodes()
    for key in ("keys", "split", "rgb"):
        assert np.array_equal(a[key], b[key]), key
    assert np.array_equal(a["dw"].view(np.uint32), b["dw"].view(np.uint32))
