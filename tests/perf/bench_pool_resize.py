#!/usr/bin/env python3
"""Brick-pool resizing (b200tsdf_resize_pool, DESIGN.md §3f) on the 100-frame 2048^3 / 10 m colour stream.

* resizePool after the stream: 2^15 -> 2^17 and 2^20 -> 2^15 (when the stream's bricks do not fit 2^15 within the load
  limit of 7/8, the smallest pool that does takes its place, and the record says so).  Wall time of the synchronous call,
  the span between CUDA events recorded on the handle's stream around it (b200tsdf_profile_begin / _end), and, from a
  separate torch.profiler pass, the kernel time of k_pool_rehash and of the fresh fill of the new pool.
* frames/s of integrateBatchDevice (batches of 20 frames, the stream resident in device memory) over the whole stream, in the
  smallest pool that fits the stream's bricks and in pools 2x and 4x that size (loads at the end of the stream of about
  0.75, 0.38 and 0.19 here: pools are powers of two), alternating the pools in every round.
Prints one JSON line and writes it to --out.

    python tests/perf/bench_pool_resize.py [--rounds 3] [--out profiles/h100_pool_resize.json]"""
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
from tests.common import frames  # noqa: E402

BATCH = 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [None] * 4


def stat(xs):
    return {"median": round(float(np.median(xs)), 3), "min": round(float(np.min(xs)), 3), "max": round(float(np.max(xs)), 3)}


def volume(pool_log2):
    cam = synth.Camera()
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, cam.cx, cam.cy); v.setIntegrateColor(True)
    v.reset()
    return v


def fuse(v, dev, poses):
    H, W = dev[0].shape[:2]
    for i in range(0, len(dev), BATCH):
        v.integrateBatchDevice([d.data_ptr() for d in dev[i:i + BATCH]], H, W, 32, poses[i:i + BATCH], rgba_off=16)
    v.sync()


def timed_resize(v, lg):
    torch.cuda.synchronize()
    v.profile_begin()
    t0 = time.perf_counter()
    v.resizePool(lg)
    wall = (time.perf_counter() - t0) * 1e3
    return wall, v.profile_end().ms_elapsed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    fr = list(frames(synth.S2, 100, stride=1, color=True, noise_seed=12345))
    poses = [p for p, _ in fr]
    dev = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for _, c in fr]
    torch.cuda.synchronize()

    big = volume(20)
    fuse(big, dev, poses)
    n = big.stats().n_bricks
    fit = 8
    while n * 8 > 7 << fit:
        fit += 1
    small = max(15, fit)
    nodes = big.download_nodes()

    # resize timings: (from, to) pairs, each round from a handle holding the stream at `from`
    pairs = [(small, max(17, small + 2)), (20, small)]
    rec = {f"{f}->{t}": {"wall_ms": [], "stream_events_ms": []} for f, t in pairs}
    for r in range(a.rounds + 1):                                      # round 0 warms up and is not recorded
        for f, t in pairs:
            big.resizePool(f)
            wall, ev = timed_resize(big, t)
            if r:
                rec[f"{f}->{t}"]["wall_ms"].append(wall); rec[f"{f}->{t}"]["stream_events_ms"].append(ev)
    after = big.download_nodes()
    same = all(np.array_equal(nodes[k].view(np.uint8), after[k].view(np.uint8)) for k in nodes)

    kernels = {}
    try:
        from torch.profiler import ProfilerActivity, profile
        for f, t in pairs:
            big.resizePool(f)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                big.resizePool(t)
                torch.cuda.synchronize()
            ks = {}
            for e in prof.events():
                for tag in ("k_pool_rehash", "k_fill_fresh"):
                    if tag in e.name:
                        ks[tag] = ks.get(tag, 0.0) + e.device_time_total / 1e3
            kernels[f"{f}->{t}"] = {k: round(x, 3) for k, x in ks.items()}
    except Exception as e:                                             # the profiler pass is extra information only
        kernels = {"error": repr(e)}

    # integrate rate against the load the pool ends the stream at
    pools = [fit, fit + 1, fit + 2]                                  # the loads a power-of-two pool can give this stream
    vols = {lg: volume(lg) for lg in pools}
    fps = {lg: [] for lg in pools}
    for r in range(a.rounds + 1):
        for lg in (pools if r % 2 == 0 else pools[::-1]):
            v = vols[lg]
            v.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fuse(v, dev, poses)
            dt = time.perf_counter() - t0
            if r:
                fps[lg].append(len(dev) / dt)
    loads = {lg: vols[lg].stats().n_bricks / (1 << lg) for lg in pools}
    name, limit, sm, sm_max = card()
    out = {"what": "resizePool and integrate rate against pool load, 100-frame 2048^3 / 10 m colour stream (640x480)",
           "gpu": name, "power_limit": limit, "sm_clock_after_run": sm, "sm_clock_max": sm_max,
           "n_bricks": int(n), "smallest_pool_log2_that_fits": int(fit), "nodes_identical_after_resizes": bool(same),
           "timing": f"ms, median and range of {a.rounds} rounds after one warm-up round; wall = host clock around the "
                     "synchronous call; stream_events = CUDA events on the handle's stream around it (includes the host "
                     "work between its launches); kernels = torch.profiler, one call",
           "resize": {k: {m: stat(x) for m, x in d.items()} for k, d in rec.items()},
           "resize_kernels_ms": kernels,
           "integrate_batch_device": {f"pool_log2={lg}": {"load_at_end": round(loads[lg], 3), "frames_per_s": stat(fps[lg])}
                                      for lg in pools}}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
