"""getVoxelCenters / getOccupiedVoxelIndices without a GPU.

tests/golden/leaf_pins.json holds digests of what the reference's own TSDFVolumeOctree::getVoxelCenters /
getOccupiedVoxelIndices return on the reference build (tools/make_leaf_pins.py, oracle/ref_leaves_capi.cpp).  The C++
restatement (oracle/tsdf_oracle_leaves.cpp: getLeaves over its pointer octree, the centres stored at split time) and the
numpy restatement over a node dump (tests/leaves.py) must reproduce them, and where oracle/_ref is built the reference's
live arrays must equal the restatement's.  The host emulation of the engine's enumeration (tests/emu/leaves_emu.cpp: the
kernels' traversal of the flat layout through the shared __host__ __device__ predicate) must equal the restatement exactly:
centre bits, index triples and order."""
import importlib.util
import json
import os

import numpy as np
import pytest

from oracle import leaves_py
from tests import leaves

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_leaf_pins", os.path.join(ROOT, "tools", "make_leaf_pins.py"))
mlp = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mlp)
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "leaf_pins.json")))


def assert_same_outputs(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k


@pytest.mark.parametrize("name", sorted(mlp.CASES))
def test_restatement_reproduces_reference_leaves(name):
    case = mlp.CASES[name]
    port = mlp.run_oracle("port", case)
    assert leaves.digest(port) == PINS["cases"][name]
    assert leaves.digest(mlp.run_dump("port", case)) == PINS["cases"][name]
    if os.path.exists(leaves_py.REF_LIB):
        assert_same_outputs(mlp.run_oracle("reference", case), port)          # the reference's own methods, live


def test_restatement_reproduces_reference_leaves_at_baseline_length():
    # the 100-frame 512^3 orbit; the 100-frame 2048^3 colour stream is replayed by the engine (tests/test_leaves_gpu.py)
    assert leaves.digest(mlp.run_oracle("port", mlp.LONG_CASES["L1_512_orbit100"])) == PINS["long_cases"]["L1_512_orbit100"]


def test_pins_cover_the_sweep_and_are_not_trivial():
    c = PINS["cases"]
    # 256^3 / 3 m: C = 3, L = 8
    assert set(c["pin_256_5_9_1"]) == {f"centers{n}" for n in (-1, 0, 1, 2, 3, 4, 7, 8, 11)} | {"occupied"}
    assert c["pin_256_5_9_1"]["centers0"][0] == 1 and c["pin_256_5_9_1"]["centers2"][0] == 64
    assert c["empty_256"]["occupied"][0] == 0 and c["empty_256"]["centers-1"][0] == 512
    for name in ("pin_256_5_9_1", "pin_512_4_13_0", "pin_2048_2_3_1", "shape_512_12m"):
        assert c[name]["occupied"][0] > 1000 and c[name]["centers-1"][0] > c[name]["occupied"][0]
    assert PINS["long_cases"]["L2_2048_color100"]["occupied"][0] > 10 ** 5


def _emu(case):
    from tests.emu.leaves_py import EmuLeavesVolume
    cfg, _, _, _, color, _, _ = case
    e = EmuLeavesVolume(integrate_color=int(color), **cfg)
    e.reset()
    return mlp.fuse(e, case)


@pytest.mark.parametrize("name", ["pin_256_5_9_1", "pin_512_4_13_0", "empty_256", "empty_512_12m", "shape_512_12m"])
def test_emulated_device_enumeration_equals_the_restatement(name):
    case = mlp.CASES[name]
    cfg = case[0]
    want = mlp.run_oracle("port", case)
    e = _emu(case)
    C, L = e.levels()[:2]
    for n in leaves.nlevels_sweep(C, L):
        got = e.leaves(n)
        assert np.array_equal(got.view(np.uint32), want[f"centers{n}"].view(np.uint32)), (name, n)
    assert np.array_equal(e.leaves(-1, occupied=True), want["occupied"])
    # and the same as restating over the emulation's own node dump
    assert leaves.digest(mlp.outputs_of(e.dump_nodes(), C, L, cfg)) == leaves.digest(want)


def test_restatement_basic_facts():
    # the root alone, the first split level, and the centre/index arithmetic of the reference
    d = {"keys": np.zeros((0, 4), np.int32), "split": np.zeros(0, np.uint8), "dw": np.zeros((0, 2), np.float32)}
    assert leaves.leaves(d, 3, 8, 3.0, 256, 0).tolist() == [[0.0, 0.0, 0.0]]
    one = leaves.leaves(d, 3, 8, 3.0, 256, 1)
    assert one.tolist()[:2] == [[-0.75, -0.75, -0.75], [-0.75, -0.75, 0.75]] and one.tolist()[4] == [0.75, -0.75, -0.75]
    assert leaves.voxel_index(3.0, 256, np.array([[-1.49, 0.0, 1.49]], np.float32)).tolist() == [[0, 128, 255]]
