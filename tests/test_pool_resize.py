"""Resizing a live volume's brick pool (b200tsdf_resize_pool, pool_rehash.cuh) on the host emulation (tests/emu/pool_emu.cpp):
the per-brick routines the kernel runs, rehash_claim and rehash_brick, move volumes of the pruning and re-splitting scenes
K1, K2, K4-K6 and the exact-tie cases E1-E5 into the smallest pool that fits and into pools of 2x and 4x that size.  After each
move every key is found within MAX_PROBE, every payload array of every brick is equal bit for bit, and every unclaimed slot
is fresh; the stream then goes on, growing the pool whenever it is more than half full, and ends on the reference's nodes.
A pool below the load limit is refused, and so is a rehash whose probe runs out, with the source untouched."""
import numpy as np
import pytest

from oracle.oracle_py import OracleVolume
from tests import dynamic_cases, general_cases
from tests.common import CFG_256, assert_same_nodes, frames
from tests.emu.pool_py import EmuPoolVolume
from cpu_tsdf_b200 import synth

# K3 is RGBNormalized, a payload the emulation does not keep
PIN_CASES = [dynamic_cases.CASES[k] for k in ("K1", "K2", "K4", "K5", "K6")] + \
            [general_cases.CASES[k] for k in ("E1", "E2", "E3", "E4", "E5")]


def smallest_fit(n):
    """the smallest pool_log2 that reset accepts whose pool holds n bricks within the 7/8 load limit"""
    lg = 8
    while n * 8 > (7 << lg):
        lg += 1
    return lg


def check_moved(e, before, lg):
    """e's pool (2^lg slots) holds exactly the claimed bricks `before` (EmuPoolVolume.claimed), bit for bit, and every other
    slot is fresh; returns e's claimed bricks"""
    assert e.capacity() == 1 << lg
    after = e.claimed()
    slots = e.find(before["keys"])
    assert (slots >= 0).all()                                   # every key within MAX_PROBE
    assert len(after["keys"]) == len(before["keys"])
    at = np.searchsorted(after["slots"], slots)
    assert np.array_equal(after["slots"][at], slots) and np.array_equal(after["keys"][at], before["keys"])
    for name in ("nodes", "split", "rgb", "M", "ns"):
        if name in before:
            assert np.array_equal(before[name].view(np.uint8), after[name][at].view(np.uint8)), name
    assert e.unclaimed_not_fresh() == 0
    return after


def same_bricks(a, b):
    return a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


def grow_at_half(e):
    """the policy INTEGRATION.md §3 recommends: double the pool while more than half of it is claimed"""
    cur = e.claimed()
    lg = int(np.log2(e.capacity()))
    while 2 * len(cur["keys"]) > (1 << lg):
        lg += 1
        assert e.resize_pool(lg) == 0
        cur = check_moved(e, cur, lg)


@pytest.mark.parametrize("case", PIN_CASES, ids=[c.id for c in PIN_CASES])
def test_pin_cases_rehash_and_continue(case):
    pool = {256: 17, 512: 18, 2048: 18, 4096: 19}[case.res]
    e = EmuPoolVolume(**case.config(), track_variance=1, pool_log2=pool); e.reset()
    o = OracleVolume(**case.config()); o.reset()
    fr = list(case.frames())
    half = max(1, len(fr) // 2)
    for pose, cloud in fr[:half]:
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    src = e.claimed()
    lg = smallest_fit(len(src["keys"]))
    cap = e.capacity()
    if lg > 8:
        assert e.resize_pool(lg - 1) == 1                           # over the load limit: refused, nothing moved
        assert e.capacity() == cap and same_bricks(src, e.claimed())
    assert e.resize_pool(lg) == 0
    raw = check_moved(e, src, lg)
    for up in (lg + 1, lg + 2):                                       # 2x and 4x the smallest pool, from it
        assert e.resize_pool(up) == 0
        check_moved(e, raw, up)
        assert e.resize_pool(lg) == 0
        raw = check_moved(e, raw, lg)
    assert e.err() == 0
    for pose, cloud in fr[half:]:
        grow_at_half(e)
        o.integrate(cloud, pose); e.integrate(cloud, pose)
        assert e.err() == 0
    assert_same_nodes(o.dump_nodes(), e.dump_nodes(), rgb=bool(case.color), var=True)


def test_probe_limit_is_reported_on_its_own_flag():
    """a rehash into a pool smaller than the brick count (the load check bypassed) runs out of probe: reported, nothing moved"""
    e = EmuPoolVolume(**CFG_256, track_variance=1, integrate_color=1, pool_log2=14); e.reset()
    for pose, cloud in frames(synth.S1, 2, stride=7, color=True, noise_seed=5):
        e.integrate(cloud, pose)
    src = e.claimed()
    assert len(src["keys"]) > 256
    assert e.resize_pool(8) == 1
    assert e.resize_pool(8, check_fit=False) == 2
    assert e.err() == 0 and e.capacity() == 1 << 14 and same_bricks(src, e.claimed())
    assert e.resize_pool(7) == 3 and e.resize_pool(27) == 3
