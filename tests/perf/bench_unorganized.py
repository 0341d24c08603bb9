#!/usr/bin/env python3
"""Unorganised clouds into the 2048^3 / 10 m colour volume: the 100-frame S2 stream of bench.py turned into unorganised clouds (every
valid pixel plus an occluded layer of 20 % of them pushed 25 % farther along their rays, shuffled), resident in device memory.
Reports, with the card's name and power limit read in the same run:

* frames/s of integrateUnorganizedBatchDevice in batches of 32, of one integrateUnorganizedCloud per frame from host memory, and of
  integrateBatchDevice in batches of 32 on the same frames organised beforehand (host clock around a pass over the 100 frames that
  ends in a sync; passes 2.. of each arm are timed, the first one captures the graphs; median over the timed passes);
* the device time of the three organise kernels per frame (torch.profiler, CUDA activities, over one batch of 32 in a run of its own).

    python tests/perf/bench_unorganized.py [--passes 4] [--out profiles/h100_unorganized.json]"""
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
from cpu_tsdf_b200 import synth  # noqa: E402
from tests.common import frames  # noqa: E402

RES, SIZE, N, BATCH = 2048, 10.0, 100, 32


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return None, None


def volume():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    cam = synth.Camera()
    v.setResolution(RES, RES, RES); v.setGridSize(SIZE, SIZE, SIZE)
    v.setCameraIntrinsics(525.0, 525.0, cam.cx, cam.cy); v.setIntegrateColor(True)
    v.reset()
    return v


def unorganized(cloud, rng):
    pts = cloud.reshape(-1, 8)
    pts = pts[~np.isnan(pts[:, 2])]
    layer = pts[rng.choice(len(pts), len(pts) // 5, replace=False)].copy()
    layer[:, :3] *= np.float32(1.25)
    allp = np.concatenate([pts, layer])
    return np.ascontiguousarray(allp[rng.permutation(len(allp))])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=4, help="passes over the stream per arm (the first is not timed)")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_unorganized.json"))
    a = ap.parse_args()
    import torch

    rng = np.random.default_rng(12345)
    stream = list(frames(synth.S2, N, stride=1, color=True, noise_seed=12345))
    poses = [p for p, _ in stream]
    clouds = [unorganized(c, rng) for _, c in stream]
    counts = [len(c) for c in clouds]
    d_clouds = [torch.from_numpy(c).cuda() for c in clouds]
    ptrs = [d.data_ptr() for d in d_clouds]
    # the same frames organised (the GPU organise, checked below against the batch's result), for the organised batch arm
    v = volume()
    organised = [v.organizeCloud(c)[0] for c in clouds]
    d_org = [torch.from_numpy(o).cuda() for o in organised]
    org_ptrs = [d.data_ptr() for d in d_org]
    torch.cuda.synchronize()
    cam = synth.Camera()

    def unorg_batches(vol):
        for k in range(0, N, BATCH):
            vol.integrateUnorganizedBatchDevice(ptrs[k:k + BATCH], counts[k:k + BATCH], 32, poses[k:k + BATCH], rgba_off=16)

    def unorg_host(vol):
        for c, p in zip(clouds, poses):
            vol.integrateUnorganizedCloud(c, p)

    def org_batches(vol):
        for k in range(0, N, BATCH):
            vol.integrateBatchDevice(org_ptrs[k:k + BATCH], cam.height, cam.width, 32, poses[k:k + BATCH], rgba_off=16)

    rec = {"what": "100-frame 2048^3 / 10 m S2 colour stream as unorganised clouds (valid pixels + a 20 % occluded layer, shuffled), "
                   "640x480 organise grid",
           "points_per_frame_mean": int(np.mean(counts)),
           "timing": f"host clock around one pass over the {N} frames ending in a sync; {a.passes} passes per arm, the first untimed, "
                     "median of the others; one fresh volume per arm"}
    nodes = {}
    for name, fn in (("unorganized_batch32", unorg_batches), ("unorganized_host_per_frame", unorg_host), ("organized_batch32", org_batches)):
        vol = volume()
        ts = []
        for i in range(a.passes):
            vol.sync()
            t0 = time.perf_counter()
            fn(vol)
            vol.sync()
            if i:
                ts.append(time.perf_counter() - t0)
        rec[f"{name}_frames_per_s"] = round(N / float(np.median(ts)), 1)
        rec[f"{name}_pass_s"] = [round(t, 4) for t in ts]
        nodes[name] = vol.download_nodes()
        del vol
    # the three arms fused the same frames the same number of times: the same volume, bit for bit
    for name in ("unorganized_host_per_frame", "organized_batch32"):
        for k in ("keys", "split", "rgb"):
            assert np.array_equal(nodes[name][k], nodes["unorganized_batch32"][k]), (name, k)
        assert np.array_equal(nodes[name]["dw"].view(np.uint32), nodes["unorganized_batch32"]["dw"].view(np.uint32)), name

    # device time of the organise kernels: one batch of 32, torch.profiler with CUDA activities
    from torch.profiler import ProfilerActivity, profile
    vol = volume()
    unorg_batches(vol); vol.sync()                                   # graphs captured outside the profiled window
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vol.integrateUnorganizedBatchDevice(ptrs[:BATCH], counts[:BATCH], 32, poses[:BATCH], rgba_off=16)
        vol.sync()
    per = {}
    for e in prof.events():
        if "k_org_" in e.name and e.device_type.name == "CUDA":
            k = "k_org_" + e.name.split("k_org_")[1].split("(")[0]
            per[k] = per.get(k, 0.0) + (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
    if per:
        rec["organize_kernels_us_per_frame"] = {k: round(t / BATCH, 2) for k, t in sorted(per.items())}
        rec["organize_us_per_frame"] = round(sum(per.values()) / BATCH, 2)
        rec["organize_timing"] = "torch.profiler (CUDA activities) over one replayed batch of 32 frames, kernel time divided by 32"
    else:
        rec["organize_us_per_frame"] = "not measured (the profiler listed no organise kernel)"
    rec["gpu"], rec["power_limit"] = card()
    print(json.dumps(rec))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
