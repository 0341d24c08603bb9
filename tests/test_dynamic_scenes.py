"""The restatement, the reference build and the host emulation on scenes that change while they are fused
(tests/dynamic_cases.py): objects shrink, vanish and come back, so pre-existing children are pruned and nodes re-split in
the same updateVoxel call.

* The restatement's outputs must reproduce the digests of the reference build's outputs stored in
  tests/golden/dynamic_pins.json (written by tools/make_dynamic_pins.py from oracle/_ref); where oracle/_ref is built, the
  reference's live outputs must reproduce them as well.  K6 pins the nodes after every frame.
* The host emulation of the engine's device code (tests/emu) must reproduce the restatement's outputs, addObservation
  counts per frame included; for K1 and K6 also with the breadth-first fresh-subtree visit at 16 records (most subtrees
  overflow into the depth-first walk) and with the recursion only.
* Every case must reach the prune events it exists for, counted by the restatement."""
import json
import os

import pytest

from oracle import oracle_py
from tests.common import digests
from tests.dynamic_cases import CASES, IDS, EmuAdapter, OracleAdapter, event_counts, outputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "dynamic_pins.json")))["dynamic_pin"]
REF_LIB = oracle_py.REF_LIB

# (pre-existing children pruned, pruned and re-split in the same call) over each stream: about 80 % of what the stream
# reaches, so that a change to the scenes cannot quietly stop driving the prune paths
FLOORS = {"K1": (4500, 140), "K2": (6800, 70), "K3": (1500, 110), "K4": (380, 60), "K5": (36000, 60), "K6": (480, 35)}

_port = {}


def port_digests(cid):
    """digests of the restatement's outputs for case `cid` (computed once per session)"""
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


# the host emulation allocates no RGBNormalized payload, so K3 is checked against the restatement on the GPU only
EMU_IDS = [cid for cid in IDS if CASES[cid].color_mode == 0]


@pytest.mark.parametrize("cid", IDS)
def test_restatement_matches_reference_pins(cid):
    got = pinned(cid, run_case(cid))
    assert "n_updates" in got


def emulation_differs(cid):
    case = CASES[cid]
    emu = digests(outputs(case, EmuAdapter(case, emu_pool_log2(case))))
    ref = port_digests(cid)
    assert emu.keys() == ref.keys()
    return [k for k in ref if emu[k] != ref[k]]


@pytest.mark.parametrize("cid", EMU_IDS)
def test_emulation_matches_restatement(cid):
    assert emulation_differs(cid) == []


@pytest.mark.parametrize("cap", ["16", "0"])
@pytest.mark.parametrize("cid", ["K1", "K6"])
def test_emulation_matches_restatement_with_other_fresh_subtree_visits(cid, cap, monkeypatch):
    """16 records: most re-split subtrees overflow the breadth-first array into the depth-first walk; 0: recursion only"""
    monkeypatch.setenv("B2_EMU_BFS_CAP", cap)
    assert emulation_differs(cid) == []


@pytest.mark.parametrize("cid", IDS)
def test_cases_reach_their_prune_events(cid):
    pruned, resplit = event_counts(CASES[cid])
    assert pruned >= FLOORS[cid][0] and resplit >= FLOORS[cid][1], (pruned, resplit)


def test_case_table_covers_what_it_is_for():
    c = CASES
    assert c["K1"].res == 256 and c["K1"].color and c["K1"].params["max_weight"] == 1.0
    assert c["K2"].res == 512 and c["K2"].track_variance and c["K2"].objects[-1].sphere is None
    assert c["K3"].color_mode == 1
    assert c["K4"].res == 2048 and c["K4"].color and len({o.box for o in c["K4"].objects}) == len(c["K4"].objects)
    assert c["K5"].res == 4096
    s6 = [o.sphere is not None for o in c["K6"].objects]
    assert s6[0] and not all(s6) and s6[-1] and c["K6"].per_frame          # present, carved, back

