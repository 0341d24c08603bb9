"""getVoxelCenters / getOccupiedVoxelIndices / isEmpty of the CUDA engine against the C++ restatement's accessors
(oracle/tsdf_oracle_leaves.cpp) and the digests of the reference's own methods (tests/golden/leaf_pins.json): arrays
compared bit for bit, order included."""
import importlib.util
import json
import os

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.leaves_py import LeavesOracleVolume as OracleVolume
from tests import leaves
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, frames

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_leaf_pins", os.path.join(ROOT, "tools", "make_leaf_pins.py"))
mlp = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mlp)
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "leaf_pins.json")))
ESTATE = -5


class Engine:
    """the Python mirror with the oracle-style integrate (cloud, pose)"""

    def __init__(self, cfg, color=False, pool_log2=18, **kw):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, **kw)
        v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
        v.setGridSize(cfg.get("xsize", 3.0), cfg.get("ysize", 3.0), cfg.get("zsize", 3.0))
        v.setCameraIntrinsics(525.0, 525.0, cfg["cx"], cfg["cy"])
        if "max_cell_x" in cfg:
            v.setMaxVoxelSize(cfg["max_cell_x"], cfg["max_cell_y"], cfg["max_cell_z"])
        v.setIntegrateColor(bool(color))
        v.reset()
        self.v = v

    def integrate(self, cloud, pose):
        self.v.integrateCloud(cloud, None, pose)

    def levels(self):
        st = self.v.stats()
        return st.coarse_level, st.finest_level

    def outputs(self):
        C, L = self.levels()
        out = {f"centers{n}": self.v.getVoxelCenters(n) for n in leaves.nlevels_sweep(C, L)}
        out["occupied"] = self.v.getOccupiedVoxelIndices()
        return out


def assert_same_outputs(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (k, got[k].shape, want[k].shape)
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k


def oracle_outputs(o):
    """getVoxelCenters / getOccupiedVoxelIndices of the C++ restatement (oracle/tsdf_oracle_leaves.cpp), checked against the
    reference's own methods in tests/test_leaves.py"""
    return mlp.method_outputs(o)


def _shape(res, size, cell):
    return dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy,
                max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)


# every shape of test_gpu_parity.py::test_other_tier_shapes, then 256^3, 512^3, 2048^3 and 4096^3
SHAPES = {
    "128_3.0_0.5": (_shape(128, 3.0, 0.5), "shape", 2, 6, False, 9, 0.0),
    "1024_3.0_0.5": (_shape(1024, 3.0, 0.5), "shape", 2, 6, False, 9, 0.0),
    "256_2.7_0.3": (_shape(256, 2.7, 0.3), "shape", 2, 6, False, 9, 0.0),
    "512_12.0_0.5": (_shape(512, 12.0, 0.5), "shape", 2, 6, False, 9, 0.0),
    "256": (CFG_256, "S1", 3, 9, True, 5, 0.0),
    "512": (CFG_512, "S1", 3, 9, False, 5, 0.0),
    "2048": (CFG_2048, "S2", 2, 3, True, 4, 0.0),
    "4096": (dict(CFG_2048, xres=4096, yres=4096, zres=4096), "S2", 1, 1, False, 4, 0.0),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_engine_leaves_equal_the_oracle(name):
    case = SHAPES[name]
    cfg, color = case[0], case[4]
    o = OracleVolume(integrate_color=int(color), **cfg); o.reset()
    e = Engine(cfg, color, pool_log2=20 if cfg["xres"] >= 2048 else 18)
    for pose, cloud in mlp.stream(case):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert e.levels() == o.levels()
    want = oracle_outputs(o)
    assert len(want["occupied"]) > 100
    assert_same_outputs(e.outputs(), want)


@pytest.mark.parametrize("name", sorted(mlp.CASES))
def test_engine_reproduces_reference_leaf_pins(name):
    case = mlp.CASES[name]
    e = mlp.fuse(Engine(case[0], case[4], pool_log2=20), case)
    assert leaves.digest(e.outputs()) == PINS["cases"][name]


@pytest.mark.parametrize("name", sorted(mlp.LONG_CASES))
def test_engine_reproduces_reference_leaf_pins_at_baseline_lengths(name):
    """the 100-frame 512^3 orbit and the 100-frame 2048^3 colour stream, every nlevels of the sweep and the occupied set"""
    case = mlp.LONG_CASES[name]
    e = mlp.fuse(Engine(case[0], case[4], pool_log2=20), case)
    assert leaves.digest(e.outputs()) == PINS["long_cases"][name]


def test_is_empty_and_leaves_across_reset_integrate_and_load(tmp_path):
    o = OracleVolume(**CFG_256); o.reset()
    e = Engine(CFG_256)
    assert e.v.isEmpty()
    assert_same_outputs(e.outputs(), oracle_outputs(o))                # an empty volume: the coarse cells only
    assert len(e.v.getVoxelCenters(-1)) == 512 and len(e.v.getOccupiedVoxelIndices()) == 0
    p_empty = str(tmp_path / "empty.vol")
    o.save(p_empty)
    for pose, cloud in frames(synth.S1, 3, stride=9, noise_seed=5):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    assert not e.v.isEmpty()
    assert e.v.getIntensityCloud() is None
    p_full = str(tmp_path / "full.vol")
    o.save(p_full)
    e.v.reset()
    assert e.v.isEmpty()
    # a .vol written by the oracle: the flag and the octree come from the file
    f = Engine(CFG_512)
    f.v.load(p_full)
    assert not f.v.isEmpty()
    assert_same_outputs(f.outputs(), oracle_outputs(o))
    f.v.load(p_empty)
    assert f.v.isEmpty()
    assert len(f.v.getVoxelCenters(-1)) == 512


def _code(exc):
    return int(str(exc.value).rsplit("(code ", 1)[1].rstrip(")"))


def test_state_errors_before_reset_and_on_a_shard():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    for call in (lambda: v.getVoxelCenters(), v.getOccupiedVoxelIndices, v.isEmpty):
        with pytest.raises(pkg.B200Error) as ei:
            call()
        assert _code(ei) == ESTATE and "before reset()" in str(ei.value)
    s = Engine(CFG_512, shard_rank=1, shard_count=2)
    for call in (lambda: s.v.getVoxelCenters(-1), s.v.getOccupiedVoxelIndices):
        with pytest.raises(pkg.B200Error) as ei:
            call()
        assert _code(ei) == ESTATE and "b200tsdf_gather_volume" in str(ei.value)
    assert s.v.isEmpty()                                             # isEmpty is per handle and allowed on a shard


def test_replica_of_two_shards_enumerates_like_the_whole_volume():
    # shards joined through export/import (the host transport of the shard gather): the replica's leaves are the volume's
    fs = list(frames(synth.S1, 4, stride=8, color=True, noise_seed=31))
    o = OracleVolume(**CFG_512, integrate_color=1); o.reset()
    full = Engine(CFG_512, True)
    for rank in range(2):
        s = Engine(CFG_512, True, shard_rank=rank, shard_count=2)
        for pose, cloud in fs:
            s.integrate(cloud, pose)
        full.v.import_shard(s.v.export_shard())
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    assert not full.v.isEmpty()
    assert_same_outputs(full.outputs(), oracle_outputs(o))
