"""The restatement, the reference build and the host emulation under general inputs (tests/general_cases.py): look-at poses
with pitch and roll, other cameras and image sizes, asymmetric truncation, sensor clipping, a non-integer weight cap, a strip
image beyond the float projection's range, exact-tie geometry and a truncation limit that makes the weighted sum overflow.

* The restatement's outputs must reproduce the digests of the reference build's outputs stored in
  tests/golden/general_pins.json (written by tools/make_general_pins.py from oracle/_ref); where oracle/_ref is built, the
  reference's live outputs must reproduce them as well.
* The host emulation of the engine's device code (tests/emu) must reproduce the restatement's outputs, addObservation
  counts per frame included.
* Case T1 must actually hit the ties it exists for."""
import json
import os

import numpy as np
import pytest

from oracle import oracle_py
from tests.common import digests
from tests.general_cases import CASES, IDS, EmuAdapter, OracleAdapter, outputs, tie_counts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "general_pins.json")))["general_pin"]
REF_LIB = oracle_py.REF_LIB

_port = {}


def port_digests(cid):
    """digests of the restatement's outputs for case `cid` (computed once per session: the pin and emulation tests share them)"""
    if cid not in _port:
        _port[cid] = digests(outputs(CASES[cid], OracleAdapter(CASES[cid])))
    return _port[cid]


def without_counts(d):
    return {k: v for k, v in d.items() if k != "n_updates"}


def run_case(cid):
    def run(kind):
        return port_digests(cid) if kind == "port" else digests(outputs(CASES[cid], OracleAdapter(CASES[cid], kind)))
    return run


def pinned(key, run):
    """run("port") must reproduce the stored digests of run("reference") (which has no addObservation counts)"""
    got = run("port")
    assert without_counts(got) == PINS[key]
    if os.path.exists(REF_LIB):
        assert run("reference") == PINS[key]
    return got


def emu_pool_log2(case):
    return 18 if case.res >= 2048 else 17


@pytest.mark.parametrize("cid", IDS)
def test_restatement_matches_reference_pins(cid):
    got = pinned(cid, run_case(cid))
    assert "n_updates" in got


@pytest.mark.parametrize("cid", IDS)
def test_emulation_matches_restatement(cid):
    case = CASES[cid]
    emu = digests(outputs(case, EmuAdapter(case, emu_pool_log2(case))))
    ref = port_digests(cid)
    assert emu.keys() == ref.keys()
    assert [k for k in ref if emu[k] != ref[k]] == []


def test_cases_reach_what_they_are_for():
    """the case table covers what tests/general_cases.py says it does"""
    for c in CASES.values():
        if c.id == "T1":
            continue
        for pose in c.poses:
            R = pose[:3, :3]
            assert abs(R[1, 1]) < 0.999 and np.abs(R[1, [0, 2]]).max() > 1e-3     # pitch or roll: the y row is not (0, 1, 0)
    assert CASES["G1"].params["max_dist_pos"] != CASES["G1"].params["max_dist_neg"]
    assert CASES["G6"].cam.width >= 8192                                            # beyond the float projection's range
    assert {CASES["G5a"].cam.width, CASES["G5b"].cam.width} == {320, 643}


def test_exact_ties_are_hit():
    """T1: axis-aligned poses with dyadic translations, walls on node planes, no noise.  Node centres in the camera frame are
    dyadic, so projections land exactly on integers and in (-1, 0), cloud points lie on node planes, and observations are
    exactly 0 or +-max_dist.  Without these counts the case could silently stop testing anything."""
    case = CASES["T1"]
    a = OracleAdapter(case)
    for pose, cloud in case.frames():
        a.integrate(cloud, pose)
    n = tie_counts(case, a.dump_nodes())
    assert n["integer_proj"] >= 100, n
    assert n["proj_in_minus1_0"] >= 100, n
    assert n["points_on_planes"] >= 100_000, n
    assert n["d_new_at_limits"] >= 1000, n


def test_division_overflow_case_reaches_inf():
    """D1: d_new / max_dist_neg is ~1e38, so the weighted sum d_old * w + d_new overflows and the reference divides inf"""
    case = CASES["D1"]
    a = OracleAdapter(case)
    for pose, cloud in case.frames():
        a.integrate(cloud, pose)
    d = a.dump_nodes()["dw"][:, 0]
    assert np.isposinf(d).sum() > 1000 and (np.abs(d) > 1e30).sum() > 100_000 and not np.isnan(d).any()
