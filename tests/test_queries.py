"""getFxn / getGradient / getHessian and getTSDFValue without a GPU, on the volumes and point sets of tests/query_cases.py.

tests/golden/query_pins.json holds digests of what the reference's own methods return on the reference build
(tools/make_query_pins.py): every point set, `what` in {1, 2, 4, 3, 7} x mode in {0, 1}, and getTSDFValue with the caller's
`valid` all true, all false and mixed.  The C++ restatement (oracle/tsdf_oracle.cpp) must reproduce them, as must the
reference build where oracle/_ref exists, and the host emulation of the device code (tests/emu: query_point and
interpolate_trilinearly as k_query and k_interpolate call them).

A float64 statement of the interpolant in numpy, which shares no code with any of them, says what the numbers mean: the
trilinear interpolant of the leaf values at the eight surrounding finest-voxel centres.  Meta-tests show that every set has
the exact ties, border layers and mixed-depth neighbourhoods it is there for."""
import functools
import json
import os

import numpy as np
import pytest

from oracle import oracle_py
from tests import query_cases as qc
from tests.common import digests
from tests.voxels import voxel_centers_1d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "query_pins.json")))["cases"]


@functools.lru_cache(maxsize=None)
def port(vid):
    """the restatement after the volume's frames, its node index and the point sets"""
    volume = qc.VOLUMES[vid]
    o = qc.OracleAdapter(volume, "port")
    nodes = o.dump_nodes()
    return o, qc.LeafIndex(nodes, volume.res), qc.point_sets(volume, nodes)


def backend_digests(vol, volume):
    nodes = vol.dump_nodes()
    return digests(qc.outputs(vol, volume, qc.point_sets(volume, nodes), qc.LeafIndex(nodes, volume.res)))


def differing(got, want):
    return [k for k in want if got.get(k) != want[k]] + [k for k in got if k not in want]


def test_pins_cover_every_volume():
    assert sorted(PINS) == sorted(qc.IDS)


@pytest.mark.parametrize("vid", qc.IDS)
def test_restatement_reproduces_reference_queries(vid):
    volume = qc.VOLUMES[vid]
    o, index, sets = port(vid)
    assert differing(digests(qc.outputs(o, volume, sets, index)), PINS[vid]) == []
    if os.path.exists(oracle_py.REF_LIB):                               # the reference's own methods, live
        assert differing(backend_digests(qc.OracleAdapter(volume, "reference"), volume), PINS[vid]) == []


@pytest.mark.parametrize("vid", qc.IDS)
def test_emulated_kernels_reproduce_reference_queries(vid):
    volume = qc.VOLUMES[vid]
    assert differing(backend_digests(qc.EmuAdapter(volume), volume), PINS[vid]) == []


def exactly_representable(volume):
    """every getVoxelCenter of the grid is the float64 value itself, so adjacent centres are exactly size / res apart"""
    s = np.float64(np.float32(volume.size))
    i = np.arange(volume.res, dtype=np.float64)
    return bool((voxel_centers_1d(volume.size, volume.res, i).astype(np.float64) == (i + 0.5) * s / volume.res - s / 2).all())


@pytest.mark.parametrize("vid", qc.IDS)
def test_queries_are_the_trilinear_interpolant_in_float64(vid):
    """At every point a call accepts: getTSDFValue and getFxn in its finest-centre form (mode 1) equal the float64 trilinear
    interpolant of the node dump to 1e-5 (the values are in [-1, 1]); away from exact centre ties, where the cell and so the
    derivative is one-sided, the mode-1 gradient equals a float64 finite difference of that interpolant to 1e-5 per voxel.
    On a grid whose centres are not floats (Q256b) adjacent rounded centres are size / res give or take an ulp of size / 2
    apart, and the reference's weights inherit that: four such ulps, in voxels, are added to both tolerances."""
    volume = qc.VOLUMES[vid]
    o, index, sets = port(vid)
    vs = volume.size / volume.res
    tol = 1e-5 if exactly_representable(volume) else 1e-5 + 4 * float(np.spacing(np.float32(volume.size / 2))) / vs
    assert exactly_representable(volume) == (vid != "Q256b")
    checked = 0
    for name in ("random", "centres", "faces", "ulp", "border", "mixed"):
        pts = sets[name]
        val, grad, _, ok = o.query(pts, 3, 1)
        f64, g64 = qc.trilinear64(index, volume.size, pts[ok], with_gradient=True)
        assert np.abs(val[ok] - f64).max() <= tol, name
        i = np.floor(qc.index_expr(volume.size, volume.res, pts[ok]))
        off_tie = (voxel_centers_1d(volume.size, volume.res, i) != pts[ok]).all(1)
        assert off_tie.sum() > 100 or name == "centres"
        assert (np.abs(grad[ok] - g64)[off_tie] * vs).max(initial=0) <= tol, name
        tv, _ = o.interpolate(pts, True)
        fin = ~np.isnan(tv)
        assert np.abs(tv[fin] - qc.trilinear64(index, volume.size, pts[fin])).max() <= tol, name
        both = ok & fin
        assert np.abs(tv[both] - val[both]).max() <= 2 * tol, name     # the two formulas are equal inside one cell
        checked += int(ok.sum()) + int(fin.sum())
    assert checked > 20000


@pytest.mark.parametrize("vid", qc.IDS)
def test_point_sets_reach_what_they_are_for(vid):
    volume = qc.VOLUMES[vid]
    o, index, sets = port(vid)
    size, res, pin = volume.size, volume.res, PINS[vid]
    for name, pts in sets.items():                                      # the pins carry the counters of these very points
        for k, v in {**qc.tie_counts(size, res, pts), **qc.border_layer_counts(size, res, pts)}.items():
            assert pin[f"{name}.{k}"] == v, (name, k)
    # exact ties: two pinned coordinates per point on average, none left once moved by an ulp
    assert pin["centres.centre"] == 2 * len(sets["centres"]) and pin["ulp.centre"] == 0
    assert pin["faces.face"] == (2 * len(sets["faces"]) if vid != "Q256b" else 226)     # 2.7 m: the faces are not floats
    assert pin["random.centre"] <= 2 and pin["mixed.centre"] <= 2                     # continuous draws
    # ties change results: on a centre, the point one ulp below takes the other cell's sign in the gradient
    c = sets["centres"]
    g = o.query(c, 2, 1)[1]
    g_dn = o.query(np.nextafter(c, np.float32(-np.inf)), 2, 1)[1]
    assert (g != g_dn).any(1).sum() > 300
    # border: both calls refuse and accept in every border layer, and differently from each other
    b = sets["border"]
    assert min(pin["border.layer0"], pin["border.layer1_2"], pin["border.layer_m3_m2"], pin["border.layer_m1"]) > 200
    assert pin["border.outside"] > 30 and pin["border.centre"] > 50 and pin["border.face"] > 50
    ok = o.query(b, 1, 0)[3]
    nan = np.isnan(o.interpolate(b, True)[0])
    assert (ok & nan).sum() > 80 and (~ok & nan).sum() > 150 and (ok & ~nan).sum() > 150 and not (~ok & ~nan).any()
    lay = np.floor(qc.index_expr(size, res, b))
    # getTSDFValue refuses the outermost voxel layers whole, getFxn only their outer halves; one layer in, both accept
    for layer, fxn, tsdf in ((0, {True, False}, {False}), (1, {True}, {True}), (res - 2, {True}, {True}), (res - 1, {True, False}, {False})):
        only = (lay == layer).any(1) & ((lay >= 2) & (lay <= res - 3) | (lay == layer)).all(1)
        assert only.sum() > 20 and set(ok[only].tolist()) == fxn and set((~nan[only]).tolist()) == tsdf, layer
    # mixed: leaves of two depths among the eight neighbours, where the leaf-centre factors of mode 0 leave [0, c]
    assert len(sets["mixed"]) >= 500 and pin["mixed.neighbourhoods_of_two_depths"] >= 500
    assert pin["mixed.neighbourhoods_of_two_depths"] == qc.mixed_depth_count(index, size, sets["mixed"])
    v0, _, _, ok0 = o.query(sets["mixed"], 1, 0)
    v1, _, _, ok1 = o.query(sets["mixed"], 1, 1)
    assert ok0.all() and ok1.all() and (v0 != v1).sum() > 400
    far = np.abs(v0 - qc.trilinear64(index, size, sets["mixed"])) > 0.05      # not an interpolation any more
    assert far.sum() > 100
    # special: nothing non-finite, beyond the grid or in the outer half of its last voxel layer is accepted, the rest is
    sp = sets["special"]
    ok = o.query(sp, 7, 1)[3]
    inside = np.isfinite(sp).all(1) & (np.abs(sp) < volume.size / 2 - size / res).all(1)
    assert pin["special.nonfinite"] >= 14 and np.array_equal(ok, inside) and 4 <= inside.sum() <= len(sp) - 14
    tv, valid = o.interpolate(sp, True)
    assert np.isnan(tv[~inside]).all() and not valid[~inside].any()
    # getTSDFValue's flag: never set by the call, cleared where a neighbour was never observed
    for name, pts in sets.items():
        assert pin[f"{name}.tsdf_none.n_valid"] == 0
        assert pin[f"{name}.tsdf_mix.n_valid"] <= pin[f"{name}.tsdf_all.n_valid"] <= len(pts) - pin[f"{name}.tsdf_all.n_nan"]
    assert 0 < pin["random.tsdf_mix.n_valid"] < pin["random.tsdf_all.n_valid"] < len(sets["random"]) - pin["random.tsdf_all.n_nan"]
