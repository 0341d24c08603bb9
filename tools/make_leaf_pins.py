#!/usr/bin/env python3
"""Generate tests/golden/leaf_pins.json from THE REFERENCE'S OWN METHODS: TSDFVolumeOctree::getVoxelCenters at a sweep of
nlevels and getOccupiedVoxelIndices, called on the reference build after each case (oracle/_ref/libcpu_tsdf_ref_leaves.so,
`make -f oracle/leaves.mk ref` where the reference tree exists), stored as [count, SHA-256] of the arrays.
tests/test_leaves.py replays the cases through the C++ restatement, the numpy restatement over the node dump and the host
emulation (CPU), tests/test_leaves_gpu.py through the CUDA engine (GPU)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cpu_tsdf_b200 import synth  # noqa: E402
from tests import leaves  # noqa: E402
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, frames  # noqa: E402

CFG_512_12M = dict(xres=512, yres=512, zres=512, xsize=12.0, ysize=12.0, zsize=12.0, cx=CAM.cx, cy=CAM.cy,
                   max_cell_x=0.5, max_cell_y=0.5, max_cell_z=0.5)          # C = 5 > L - 6 = 3: two levels above C in the top brick

# name -> (config, scene, frames, stride, colour, noise seed, dropout)
CASES = {
    # the INTEGRATE configurations of tests/test_ref_pin.py
    "pin_256_5_9_1": (CFG_256, "S1", 5, 9, True, 7, 0.01),
    "pin_512_4_13_0": (CFG_512, "S1", 4, 13, False, 7, 0.01),
    "pin_2048_2_3_1": (CFG_2048, "S2", 2, 3, True, 7, 0.01),
    # straight after reset(): nothing below the coarse cells
    "empty_256": (CFG_256, "S1", 0, 1, False, None, 0.0),
    "empty_512_12m": (CFG_512_12M, "S1", 0, 1, False, None, 0.0),
    # a shape whose coarse cells lie inside the top-tier bricks (the frames of tests/test_gpu_parity.py::test_other_tier_shapes)
    "shape_512_12m": (CFG_512_12M, "shape", 2, 6, False, 9, 0.0),
}
# BASELINE.json lengths (tools/make_golden.py LONG_CASES): the 100-frame 512^3 orbit and the 100-frame 2048^3 colour stream
LONG_CASES = {
    "L1_512_orbit100": (CFG_512, "S1", 100, 1, False, 2, 0.0),
    "L2_2048_color100": (CFG_2048, "S2", 100, 1, True, 12345, 0.0),
}


def scene_of(name, cfg):
    if name == "shape":
        return synth.Scene(room_half=min(1.3, cfg["xsize"] * 0.45), cam_radius=0.8)
    return getattr(synth, name)


def stream(case):
    cfg, scene, n, stride, color, noise, dropout = case
    return frames(scene_of(scene, cfg), n, stride=stride, color=color, noise_seed=noise, dropout=dropout)


def fuse(vol, case):
    """integrate the case's frames into `vol` (oracle-style integrate (cloud, pose))"""
    for pose, cloud in stream(case):
        vol.integrate(cloud, pose)
    return vol


def outputs_of(dump, coarse, finest, cfg):
    """the numpy restatement (tests/leaves.py) over a node dump"""
    return leaves.leaf_outputs(dump, coarse, finest, cfg.get("xsize", 3.0), cfg["xres"])


def oracle_volume(kind, case):
    """oracle `kind` ("port" = the C++ restatement, "reference" = oracle/_ref) with the accessors, after the case's frames"""
    from oracle.leaves_py import LeavesOracleVolume
    cfg, _, _, _, color, _, _ = case
    v = LeavesOracleVolume(kind=kind, integrate_color=int(color), **cfg)
    v.reset()
    return fuse(v, case)


def method_outputs(v):
    """getVoxelCenters (every nlevels of the sweep) and getOccupiedVoxelIndices as the oracle's own methods return them"""
    coarse, finest = v.levels()
    out = {f"centers{n}": v.voxel_centers(n) for n in leaves.nlevels_sweep(coarse, finest)}
    out["occupied"] = v.occupied_voxel_indices()
    return out


def run_oracle(kind, case):
    return method_outputs(oracle_volume(kind, case))


def run_dump(kind, case):
    """the numpy restatement over the node dump of oracle `kind`"""
    v = oracle_volume(kind, case)
    coarse, finest = v.levels()
    return outputs_of(v.dump_nodes(), coarse, finest, case[0])


def main():
    from oracle import leaves_py
    if not os.path.exists(leaves_py.REF_LIB):
        raise SystemExit("oracle/_ref/libcpu_tsdf_ref_leaves.so is not built: run `make -f oracle/leaves.mk ref` where the reference tree exists")
    out = {"generator": "tools/make_leaf_pins.py",
           "source": "TSDFVolumeOctree::getVoxelCenters / getOccupiedVoxelIndices of oracle/_ref = the reference's src/lib/*.cpp "
                     "compiled verbatim (sdmiller/cpu_tsdf @ 9b973cb), called through oracle/ref_leaves_capi.cpp",
           "cases": {k: leaves.digest(run_oracle("reference", c)) for k, c in CASES.items()},
           "long_cases": {k: leaves.digest(run_oracle("reference", c)) for k, c in LONG_CASES.items()}}
    path = os.path.join(ROOT, "tests", "golden", "leaf_pins.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", path)
    for group in ("cases", "long_cases"):
        for k, v in out[group].items():
            print(k, {a: b[0] for a, b in v.items()})


if __name__ == "__main__":
    main()
