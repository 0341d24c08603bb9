#!/usr/bin/env python3
"""Leaf enumeration time: getOccupiedVoxelIndices and getVoxelCenters (-1) after the 100-frame 2048^3 colour stream
(tools/make_golden.py L2_2048_color100), on the GPU (wall time of the synchronous call: counting pass, emitting pass, radix
sort, copy to the host) beside the same calls on the CPU of the same machine: the reference's own
TSDFVolumeOctree::getOccupiedVoxelIndices / getVoxelCenters (oracle/_ref/libcpu_tsdf_ref_leaves.so, where it is built) and
the C++ restatement's (oracle/libtsdf_oracle_leaves.so), both single-threaded recursive walks of a pointer octree.  Prints
one JSON line with the leaf counts, the card's name and power limit.

    python tests/perf/bench_leaves.py [--repeats 5] [--no-cpu]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import cpu_tsdf_b200 as pkg  # noqa: E402
from tests.common import frames  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return None, None


def timed(fn, repeats):
    ts, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    cfg = dict(xres=2048, yres=2048, zres=2048, xsize=10.0, ysize=10.0, zsize=10.0)
    stream = list(frames(synth.S2, 100, stride=1, color=True, noise_seed=12345))
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, synth.Camera().cx, synth.Camera().cy); v.setIntegrateColor(True)
    v.reset()
    for pose, cloud in stream:
        v.integrateCloud(cloud, None, pose)
    v.sync()
    v.getOccupiedVoxelIndices(); v.getVoxelCenters(-1)                 # warm-up (module load, first allocations)
    ms_occ, occ = timed(v.getOccupiedVoxelIndices, a.repeats)
    ms_all, allc = timed(lambda: v.getVoxelCenters(-1), a.repeats)
    name, limit = card()
    rec = {"what": "leaf enumeration after the 100-frame 2048^3 colour stream", "gpu": name, "power_limit": limit,
           "n_leaves": int(len(allc)), "n_occupied": int(len(occ)),
           "gpu_ms_getOccupiedVoxelIndices": round(ms_occ, 3), "gpu_ms_getVoxelCenters_all": round(ms_all, 3),
           "gpu_timing": f"wall time of the synchronous call, median of {a.repeats}"}
    if not a.no_cpu:
        from oracle import leaves_py
        kinds = ["port"] + (["reference"] if os.path.exists(leaves_py.REF_LIB) else [])
        for kind in kinds:
            o = leaves_py.LeavesOracleVolume(kind=kind, integrate_color=1, cx=synth.Camera().cx, cy=synth.Camera().cy, **cfg)
            o.reset()
            for pose, cloud in stream:
                o.integrate(cloud, pose)
            ms_cocc, cocc = timed(o.occupied_voxel_indices, 1)
            ms_call, call = timed(lambda: o.voxel_centers(-1), 1)
            assert np.array_equal(cocc, occ) and np.array_equal(call.view(np.uint32), allc.view(np.uint32))
            name_ = "cpu_reference" if kind == "reference" else "cpu_restatement"
            rec.update({f"{name_}_ms_getOccupiedVoxelIndices": round(ms_cocc, 1), f"{name_}_ms_getVoxelCenters_all": round(ms_call, 1)})
            del o
        rec["cpu"] = ("same machine, one run each: cpu_reference = the reference's own methods (oracle/_ref), cpu_restatement = "
                      "oracle/tsdf_oracle_leaves.cpp; both return the same arrays as the GPU")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
