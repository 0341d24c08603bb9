#!/usr/bin/env python3
"""Dense crop and point lookup time after the 100-frame 2048^3 colour stream (tools/make_golden.py L2_2048_color100).

* k_dense: a 512^3 crop centred on the occupied leaves, all four outputs (d, w float32; rgb 3 B; level 1 B: 12 B per voxel).
* the same crop as point lookups: b200tsdf_containing_voxels_device on the 512^3 voxel centres (44-byte records), alternated
  with k_dense in one process; the fields they share are checked equal once.
* point lookups of 10 M uniform points in the volume.

Wall time: host clock around the call and a synchronise of the handle's stream, medians and ranges over alternated rounds.
Device time: the kernels' durations under torch.profiler in a separate pass.  Output bytes per second are the bytes the box
implies over device time, beside the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line with the card's name and power
limit, read in the same run.

    python tests/perf/bench_voxels.py [--rounds 7] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import cpu_tsdf_b200 as pkg  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402
from tests import voxels  # noqa: E402
from tests.common import frames  # noqa: E402

HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return [s.strip() for s in q.split(",")]


def wall(fn, v):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    v.sync()
    return (time.perf_counter() - t0) * 1e3


def device_ms(fn, v, name, reps=5):
    """mean duration of the kernels whose name contains `name`, per call, under torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        v.sync()
        torch.cuda.synchronize()
    tot = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
    return tot / reps / 1e3


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3), "max_ms": round(float(np.max(ts)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit, clock = card()
    res, size = 2048, 10.0
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    v.setResolution(res, res, res); v.setGridSize(size, size, size)
    v.setCameraIntrinsics(525.0, 525.0, synth.Camera().cx, synth.Camera().cy); v.setIntegrateColor(True)
    v.reset()
    for pose, cloud in frames(synth.S2, 100, stride=1, color=True, noise_seed=12345):
        v.integrateCloud(cloud, None, pose)
    v.sync()
    occ = v.getOccupiedVoxelIndices()
    c = np.median(occ, axis=0).astype(int)
    lo = np.clip(c - 256, 0, res - 512)
    box = (int(lo[0]), int(lo[1]), int(lo[2]), int(lo[0]) + 512, int(lo[1]) + 512, int(lo[2]) + 512)
    n = 512 ** 3
    dev = "cuda"
    d = torch.empty(n, dtype=torch.float32, device=dev); w = torch.empty(n, dtype=torch.float32, device=dev)
    rgb = torch.empty(3 * n, dtype=torch.uint8, device=dev); lvl = torch.empty(n, dtype=torch.int8, device=dev)
    axes = [torch.from_numpy(voxels.voxel_centers_1d(size, res, np.arange(box[k], box[k + 3]))).to(dev) for k in range(3)]
    pts = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3).contiguous()
    rec = torch.empty(44 * n, dtype=torch.uint8, device=dev)
    dense = lambda: v.extractDenseDevice(box, d.data_ptr(), w.data_ptr(), rgb.data_ptr(), lvl.data_ptr())
    look = lambda: v.getContainingVoxelsDevice(pts.data_ptr(), n, rec.data_ptr())
    dense(); look(); v.sync()
    r = rec.view(-1, 44)
    same = (torch.equal(r[:, 32:36].contiguous().view(torch.float32).view(-1), d) and torch.equal(r[:, 36:40].contiguous().view(torch.float32).view(-1), w)
            and torch.equal(r[:, 40:43].reshape(-1), rgb) and torch.equal(r[:, 0].to(torch.int8), lvl))
    assert same, "k_dense and the lookups at the voxel centres differ"
    del r
    td, tl = [], []
    for _ in range(a.rounds):
        td.append(wall(dense, v)); tl.append(wall(look, v))
    dev_dense = device_ms(dense, v, "k_dense")
    dev_look = device_ms(look, v, "k_voxels")
    del pts, rec
    torch.cuda.empty_cache()
    m = 10_000_000
    up = torch.from_numpy(np.random.default_rng(0).uniform(-5.0, 5.0, (m, 3)).astype(np.float32)).to(dev)
    urec = torch.empty(44 * m, dtype=torch.uint8, device=dev)
    ulook = lambda: v.getContainingVoxelsDevice(up.data_ptr(), m, urec.data_ptr())
    ulook(); v.sync()
    tu = [wall(ulook, v) for _ in range(a.rounds)]
    dev_u = device_ms(ulook, v, "k_voxels")
    out_bytes = 12 * n
    out = {"what": "dense crop and point lookups after the 100-frame 2048^3 colour stream", "gpu": name, "power_limit": limit,
           "max_sm_clock": clock, "box": list(box), "voxels": n, "n_occupied_leaves": int(len(occ)),
           "dense_k_dense": dict(stats(td), device_ms=round(dev_dense, 3), output_bytes=out_bytes,
                                 output_TBps=round(out_bytes / (dev_dense * 1e-3) / 1e12, 3),
                                 share_of_3_35_TBps=round(out_bytes / (dev_dense * 1e-3) / 1e12 / HBM_TBS, 3)),
           "dense_as_lookups_k_voxels": dict(stats(tl), device_ms=round(dev_look, 3), input_bytes=12 * n, output_bytes=44 * n),
           "lookups_10M_uniform": dict(stats(tu), device_ms=round(dev_u, 3), lookups_per_s=round(m / (dev_u * 1e-3), 0)),
           "timing": f"wall: host clock around call + stream sync, {a.rounds} rounds, the two crop arms alternated; device: "
                     "torch.profiler kernel durations, mean of 5 calls",
           "fields_equal": bool(same)}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
