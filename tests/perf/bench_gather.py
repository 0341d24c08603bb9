#!/usr/bin/env python3
"""Where a frame of the bench workload goes on the device, and how much the pixel gather costs.

The workload is bench.py's headline leg: the same 64 synthetic 640x480 S2 frames, colour on, 2048^3 / 10 m,
integrateBatchDevice with 32 frames per call (one graph launch), warmed up the same way.  Two parts:

  split      mean device time per frame of k_front, k_celltop_down, k_bricks and k_celltop_up under torch.profiler
             (CUDA activities; kernels inside the replayed graphs are recorded one by one).  The kernels are linked by
             programmatic dependent launch, so a kernel's blocks start while its predecessor drains and wait for it: `span`
             (first block start -> last block end) counts that wait, `adds` (its end minus the predecessor's end) is what the
             kernel adds to the frame.  The gap is the frame time of an unprofiled run minus the sum of the four `adds`.
  footprint  the same stream from clouds repacked on the host to 16-byte points {x, y, z, bgra} (stride 16) against the
             32-byte points bench.py feeds (stride 32), alternated in one process, `--repeats` runs each.  Every run starts
             from reset() and repeats bench.py's warm-up, so both layouts fuse exactly the same frames into the same state.

Beside the times it prints the last frame's stats() counters (n_culled_cells, n_node_visits) and the card's name, power
limit and clocks.  One JSON line on stdout; `--out FILE` writes it there as well.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload's inputs and constants; bench.main is not run)

FOUR = ("k_front", "k_celltop_down", "k_bricks", "k_celltop_up")
KERNEL_RE = re.compile(r"\b(k_[A-Za-z0-9_]+)")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [c.strip() for c in r.stdout.strip().split(",")]))
    except Exception as e:            # no nvidia-smi: the torch name alone
        import torch
        return {"name": torch.cuda.get_device_name(0), "error": type(e).__name__}


def repack16(c32):
    """[H, W, 8] float32 points (x, y, z, pad, bgra at byte 16, ...) -> [H, W, 4] {x, y, z, bgra}: the same bits."""
    return np.ascontiguousarray(c32[:, :, [0, 1, 2, 4]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=4)
    ap.add_argument("--out")
    args = ap.parse_args()

    import torch
    import cpu_tsdf_b200 as pkg
    from cpu_tsdf_b200.build import build_library
    build_library()
    torch.cuda.set_device(0)
    F = bench.FRAMES_PER_STEP
    ND = bench.N_DISTINCT
    poses, clouds = bench.make_inputs()
    layouts = {32: ([torch.from_numpy(c).cuda() for c in clouds], 16),
               16: ([torch.from_numpy(repack16(c)).cuda() for c in clouds], 12)}
    vol = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
    vol.setGridSize(bench.SIZE, bench.SIZE, bench.SIZE)
    vol.setResolution(bench.RES, bench.RES, bench.RES)
    vol.setCameraIntrinsics(bench.CAM.fx, bench.CAM.fy, bench.CAM.cx, bench.CAM.cy)
    vol.setIntegrateColor(True)

    def step(stride, k0):
        d, roff = layouts[stride]
        idx = [(k0 + j) % ND for j in range(F)]
        vol.integrateBatchDevice([d[i].data_ptr() for i in idx], bench.H, bench.W, stride, [poses[i] for i in idx], rgba_off=roff)

    def warm(stride):
        vol.reset()
        k = 0
        for _ in range(args.warmup):
            step(stride, k); k += F
        vol.sync()
        return k

    def timed_run(stride):
        k = warm(stride)
        vol.profile_begin()
        for _ in range(args.steps):
            step(stride, k); k += F
        pr = vol.profile_end()
        vol.sync()
        st = vol.stats()
        n = args.steps * F
        return {"frames_per_s": n / (pr.ms_elapsed / 1e3), "us_per_frame": 1e3 * pr.ms_elapsed / n,
                "k_bricks_us_device_timer": 1e3 * pr.ms_kernel_device / max(1, pr.kernel_launches_device),
                "node_visits_per_frame": pr.n_node_visits / max(1, pr.n_frames), "updates_per_frame": pr.n_updates / max(1, pr.n_frames),
                "last_frame": {"n_culled_cells": int(st.n_culled_cells), "n_node_visits": int(st.n_node_visits),
                               "n_block_visits": int(st.n_block_visits), "n_updates": int(st.n_updates)}}

    def split(stride, frame_us):
        from torch.profiler import ProfilerActivity, profile
        k = warm(stride)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                step(stride, k); k += F
            vol.sync()
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "trace.json")
            prof.export_chrome_trace(path)
            trace = json.load(open(path))
        n = args.profile_steps * F
        ev = []
        for e in trace.get("traceEvents", []):
            if e.get("cat") != "kernel":
                continue
            m = KERNEL_RE.search(e.get("name", ""))
            ev.append((float(e["ts"]), float(e.get("dur", 0.0)), m.group(1) if m else e.get("name", "")[:60]))
        ev.sort()
        # span: first block start -> last block end, including the time its blocks wait on griddepcontrol.wait for the
        # predecessor; adds: how far the kernel moves the end of the chain (its end minus the predecessor's end)
        tot, add, cnt = {}, {}, {}
        prev_end = None
        for ts, dur, nm in ev:
            tot[nm] = tot.get(nm, 0.0) + dur
            cnt[nm] = cnt.get(nm, 0) + 1
            end = ts + dur
            add[nm] = add.get(nm, 0.0) + (end - prev_end if prev_end is not None else dur)
            prev_end = end if prev_end is None else max(prev_end, end)
        per = {nm: {"span_us_per_frame": tot[nm] / n, "adds_us_per_frame": add[nm] / n, "launches_per_frame": cnt[nm] / n}
               for nm in sorted(tot, key=lambda x: -add[x])}
        four_span = sum(per[nm]["span_us_per_frame"] for nm in FOUR if nm in per)
        four_add = sum(per[nm]["adds_us_per_frame"] for nm in FOUR if nm in per)
        return {"kernels": per, "sum_of_four_span_us": four_span, "sum_of_four_adds_us": four_add,
                "frame_us_unprofiled": frame_us, "gap_us": frame_us - four_add,
                "frame_us_profiled": (prev_end - ev[0][0]) / n if ev else None, "frames_profiled": n}

    out = {"card_before": card(), "workload": "bench.py headline leg: 64 S2 frames 640x480, colour on, 2048^3 / 10 m, integrateBatchDevice x32",
           "steps": args.steps, "warmup": args.warmup}
    runs = {16: [], 32: []}
    timed_run(32)                      # one discarded run: first graph captures, clocks settling
    for _ in range(args.repeats):
        for stride in (32, 16):
            runs[stride].append(timed_run(stride))
    out["footprint"] = {}
    for stride, rs in runs.items():
        fps = [r["frames_per_s"] for r in rs]
        kb = [r["k_bricks_us_device_timer"] for r in rs]
        out["footprint"][f"stride{stride}"] = {"frames_per_s": fps, "frames_per_s_median": float(np.median(fps)),
                                               "spread_pct": 100.0 * (max(fps) - min(fps)) / float(np.median(fps)),
                                               "k_bricks_us": kb, "k_bricks_us_median": float(np.median(kb)), "runs": rs}
    out["split"] = {f"stride{s}": split(s, float(np.median([r["us_per_frame"] for r in runs[s]]))) for s in (32, 16)}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
