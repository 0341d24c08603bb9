#!/usr/bin/env python3
"""Tracking (DESIGN.md §3i) after the 100-frame 2048^3 / 10 m colour stream of bench.py (S2 orbit, 640x480, fused from uint16
depth maps).  Reports, with the card's name, power limit and SM clocks read in the same run:

* wall time per trackDepth call (host depth map, default schedule, start 1 cm / 0.5 deg off the ground truth): host clock
  around each call (the call returns with its result on the host), median and spread over every frame of every round;
* device time per call and its split between k_depth_unproject, k_track_terms and k_track_solve: torch.profiler with CUDA
  activities, one pass over the 100 frames in a run of its own;
* frames/s of the track-then-integrate loop from host depth maps (trackDepth from the previous estimate, then integrateDepth
  with the result), over the 100 frames into a fresh volume seeded with frame 0;
* the CPU arm: the same schedule on the host emulation of track.cuh (one thread) and on the device, on a 512^3 / 3 m volume of
  ten S1 frames (the emulation cannot hold the 2048^3 volume), the same held-out frames for both.  The reference has no
  tracker, so this is the only CPU comparison there is.

    python tests/perf/bench_track.py [--rounds 3] [--out profiles/h100_track.json]"""
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
from tests.test_depth_images import depth_frame  # noqa: E402

RES, SIZE, N = 2048, 10.0, 100


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [None] * 4


def nudge(pose, k):
    """the start pose of frame k: 1 cm and 0.5 deg off, in a direction that changes with k"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(k)
    d = np.eye(4)
    a = rng.standard_normal(3); a *= np.radians(0.5) / np.linalg.norm(a)
    t = rng.standard_normal(3); t *= 0.01 / np.linalg.norm(t)
    d[:3, :3] = Rotation.from_rotvec(a).as_matrix(); d[:3, 3] = t
    return d @ pose


def volume(res=RES, size=SIZE, color=True, pool=20):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool)
    cam = synth.Camera()
    v.setResolution(res, res, res); v.setGridSize(size, size, size)
    v.setCameraIntrinsics(525.0, 525.0, cam.cx, cam.cy); v.setIntegrateColor(color)
    v.reset()
    return v


def stats(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(ts)), "p10_ms": float(np.percentile(ts, 10)), "p90_ms": float(np.percentile(ts, 90)),
            "min_ms": float(ts.min()), "max_ms": float(ts.max()), "n": int(len(ts))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_track.json"))
    a = ap.parse_args()
    import torch

    stream = list(frames(synth.S2, N, stride=1, color=True, noise_seed=12345))
    poses = [p for p, _ in stream]
    depths, rgbs = zip(*[depth_frame(c) for _, c in stream])
    v = volume()
    for p, d, c in zip(poses, depths, rgbs):
        v.integrateDepth(d, p, c, 1e-3)
    v.sync()
    starts = [nudge(p, k) for k, p in enumerate(poses)]
    prm = pkg.TrackParams.default()

    # wall time per call (round 0 captures the graph and is not timed)
    wall, status, errs = [], [], []
    for r in range(a.rounds + 1):
        for k in range(N):
            t0 = time.perf_counter()
            pose, res = v.trackDepth(depths[k], starts[k], prm, 1e-3)
            t1 = time.perf_counter()
            if r:
                wall.append(t1 - t0)
            if r == 1:
                status.append(res["status"]); errs.append(float(np.linalg.norm(pose[:3, 3] - poses[k][:3, 3])))

    # device time and split, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(N):
            v.trackDepth(depths[k], starts[k], prm, 1e-3)
    split = {}
    for e in prof.key_averages():
        for name in ("k_track_terms", "k_track_solve", "k_depth_unproject"):
            if name in e.key:
                split[name] = split.get(name, 0.0) + e.device_time_total / 1e3 / N        # ms per call
    device_ms = sum(split.values())

    # track-then-integrate loop
    loop = []
    for r in range(a.rounds):
        w = volume()
        w.integrateDepth(depths[0], poses[0], rgbs[0], 1e-3)
        est = poses[0]
        w.sync()
        t0 = time.perf_counter()
        for k in range(1, N):
            est, _ = w.trackDepth(depths[k], est, prm, 1e-3)
            w.integrateDepth(depths[k], est, rgbs[k], 1e-3)
        w.sync()
        loop.append((N - 1) / (time.perf_counter() - t0))
        drift = float(np.linalg.norm(est[:3, 3] - poses[-1][:3, 3]))
        del w

    # the CPU arm: host emulation (one thread) against the device on one 512^3 / 3 m S1 volume
    from tests.emu import track_py
    cam = synth.Camera()
    e = track_py.TrackEmuVolume(xres=512, yres=512, zres=512, cx=cam.cx, cy=cam.cy, pool_log2=17)
    e.reset()
    g = volume(512, 3.0, False, 17)
    for f in range(0, 100, 10):
        p = synth.orbit_pose(synth.S1, f, 100)
        c = synth.make_frame(synth.S1, p, cam, noise_seed=3, frame=f)
        e.integrate(c, p); g.integrateCloud(c, None, p)
    held = [(synth.orbit_pose(synth.S1, f, 100), synth.make_frame(synth.S1, synth.orbit_pose(synth.S1, f, 100), cam)) for f in (5, 25, 45)]
    emu_t, dev_t = [], []
    for k, (p, c) in enumerate(held):
        d16 = depth_frame(np.concatenate([c, np.zeros(c.shape[:2] + (4,), np.float32)], -1))[0]
        g.trackDepth(d16, nudge(p, k), prm, 1e-3)                          # capture
        t0 = time.perf_counter(); e.track(d16, nudge(p, k), prm); emu_t.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); g.trackDepth(d16, nudge(p, k), prm, 1e-3); dev_t.append(time.perf_counter() - t0)

    name, limit, clk, clk_max = card()
    out = {
        "card": name, "power_limit": limit, "sm_clock_at_end": clk, "sm_clock_max": clk_max,
        "workload": f"{N}-frame S2 colour orbit fused into {RES}^3 / {SIZE} m from uint16 depth maps, 640x480; default schedule "
                    f"(levels {prm.levels}, strides {list(prm.stride)[:prm.levels]}, iters {list(prm.iters)[:prm.levels]})",
        "track_call_wall": stats(wall),
        "track_call_device_ms": device_ms,
        "device_split_ms_per_call": split,
        "status_counts": {str(s): status.count(s) for s in sorted(set(status))},
        "translation_error_m": {"median": float(np.median(errs)), "max": float(np.max(errs))},
        "track_then_integrate_fps": {"median": float(np.median(loop)), "all": loop, "final_drift_m": drift},
        "cpu_arm_512_s1": {"host_emulation_one_thread": stats(emu_t), "device": stats(dev_t),
                           "note": "host emulation of track.cuh, one thread; the reference has no tracker"},
    }
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
