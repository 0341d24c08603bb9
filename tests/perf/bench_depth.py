#!/usr/bin/env python3
"""Depth images into the 2048^3 / 10 m colour volume: the 100-frame S2 colour orbit of bench.py at 640x480 as uint16 depth maps
(z in mm, NaN -> 0) with registered RGB8 images, against the same frames as depth_to_cloud clouds.  Reports, with the card's name
and power limit read in the same run:

* end to end from pinned host memory: frames/s of integrateDepth (one call per frame, uint16 + RGB8) against bench.py's
  end-to-end route (integrateBatchRows on one GPU, 32-byte points in batches of 32) and one integrateCloud per frame;
* device-resident: frames/s of integrateDepthBatchDevice against integrateBatchDevice on the depth_to_cloud clouds, 32 frames
  per call;
* the device time of k_depth_unproject per frame (torch.profiler, CUDA activities, one replayed batch of 32 in a run of its
  own) and its bytes per second (2 B depth + 3 B colour read, 16 B written per pixel) against the data sheet's 3.35 TB/s.

Rates: host clock around a pass over the 100 frames that ends in a sync; the arms alternate round by round on one volume each,
round 0 (graph capture) is not timed, the median of the others is reported.

    python tests/perf/bench_depth.py [--rounds 5] [--out profiles/h100_depth.json]"""
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
from cpu_tsdf_b200 import DEPTH_U16, depth_to_cloud, synth  # noqa: E402
from tests.common import frames  # noqa: E402
from tests.test_depth_images import depth_frame  # noqa: E402

RES, SIZE, N, BATCH = 2048, 10.0, 100, 32
HBM_BYTES_PER_S = 3.35e12                                   # H100 SXM data sheet


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="rounds over the arms (round 0 is not timed)")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_depth.json"))
    a = ap.parse_args()
    import torch

    cam = synth.Camera()
    W, H = cam.width, cam.height
    intr = (525.0, 525.0, cam.cx, cam.cy)
    stream = list(frames(synth.S2, N, stride=1, color=True, noise_seed=12345))
    poses = [p for p, _ in stream]
    depths, rgbs = zip(*[depth_frame(c) for _, c in stream])
    clouds = [depth_to_cloud(d, intr, c, 1e-3) for d, c in zip(depths, rgbs)]
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    h_depth = [pin(d) for d in depths]
    h_rgb = [pin(c) for c in rgbs]
    h_cloud = [pin(c) for c in clouds]
    n_depth = [t.numpy() for t in h_depth]
    n_rgb = [t.numpy() for t in h_rgb]
    n_cloud = [t.numpy() for t in h_cloud]
    d_depth = [t.cuda() for t in h_depth]
    d_rgb = [t.cuda() for t in h_rgb]
    d_cloud = [t.cuda() for t in h_cloud]
    torch.cuda.synchronize()
    dp = lambda ts: [t.data_ptr() for t in ts]

    def depth_host(v):
        for d, c, p in zip(n_depth, n_rgb, poses):
            v.integrateDepth(d, p, c, 1e-3)

    def rows_host(v):
        for k in range(0, N, BATCH):
            v.integrateBatchRows(dp(h_cloud[k:k + BATCH]), H, W, 32, poses[k:k + BATCH], rgba_off=16)

    def cloud_host(v):
        for c, p in zip(n_cloud, poses):
            v.integrateCloud(c, None, p)

    def depth_device(v):
        for k in range(0, N, BATCH):
            v.integrateDepthBatchDevice(dp(d_depth[k:k + BATCH]), poses[k:k + BATCH], depth_format=DEPTH_U16, depth_scale=1e-3,
                                        d_rgb_ptrs=dp(d_rgb[k:k + BATCH]))

    def cloud_device(v):
        for k in range(0, N, BATCH):
            v.integrateBatchDevice(dp(d_cloud[k:k + BATCH]), H, W, 32, poses[k:k + BATCH], rgba_off=16)

    arms = {"e2e_integrate_depth": depth_host, "e2e_batch_rows_32B": rows_host, "e2e_integrate_cloud_32B": cloud_host,
            "device_depth_batch32": depth_device, "device_cloud_batch32": cloud_device}
    rec = {"what": "100-frame 2048^3 / 10 m S2 colour orbit at 640x480: uint16 depth (mm) + RGB8 against the same frames as "
                   "depth_to_cloud clouds (32-byte points)",
           "bytes_per_frame": {"depth_u16_rgb8": W * H * 5, "cloud_32B": W * H * 32},
           "timing": f"host clock around one pass over the {N} frames ending in a sync; {a.rounds} rounds with the arms alternated, "
                     "round 0 untimed, median of the others; one volume per arm, not reset between rounds"}
    vols = {}
    ts = {k: [] for k in arms}
    for r in range(a.rounds):
        for name, fn in arms.items():
            if name not in vols:
                vols[name] = volume()
            v = vols[name]
            v.sync()
            t0 = time.perf_counter()
            fn(v)
            v.sync()
            if r:
                ts[name].append(time.perf_counter() - t0)
        if r == 0:
            # every arm fused the same frames once: the same volume, bit for bit
            ref = vols["e2e_batch_rows_32B"].download_nodes()
            for name, v in vols.items():
                got = v.download_nodes()
                for k in ("keys", "split", "rgb"):
                    assert np.array_equal(got[k], ref[k]), (name, k)
                assert np.array_equal(got["dw"].view(np.uint32), ref["dw"].view(np.uint32)), name
            rec["same_volume_after_round0"] = True
    for name in arms:
        rec[f"{name}_frames_per_s"] = round(N / float(np.median(ts[name])), 1)
        rec[f"{name}_pass_s"] = [round(t, 4) for t in ts[name]]
    vols.clear()

    from torch.profiler import ProfilerActivity, profile
    v = volume()
    depth_device(v); v.sync()                                        # graphs captured outside the profiled window
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        v.integrateDepthBatchDevice(dp(d_depth[:BATCH]), poses[:BATCH], depth_format=DEPTH_U16, depth_scale=1e-3,
                                    d_rgb_ptrs=dp(d_rgb[:BATCH]))
        v.sync()
    us = n = 0
    for e in prof.events():
        if "k_depth_unproject" in e.name and e.device_type.name == "CUDA":
            us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            n += 1
    if n:
        per = us / BATCH
        rec["k_depth_unproject_us_per_frame"] = round(per, 3)
        rec["k_depth_unproject_launches"] = n
        bytes_frame = W * H * (2 + 3 + 16)
        rec["k_depth_unproject_bytes_per_frame"] = bytes_frame
        rec["k_depth_unproject_TB_per_s"] = round(bytes_frame / (per * 1e-6) / 1e12, 3)
        rec["k_depth_unproject_share_of_3.35TB_per_s"] = round(bytes_frame / (per * 1e-6) / HBM_BYTES_PER_S, 3)
        rec["k_depth_unproject_timing"] = "torch.profiler (CUDA activities) over one replayed batch of 32 frames, kernel time / 32"
    else:
        rec["k_depth_unproject_us_per_frame"] = "not measured (the profiler listed no k_depth_unproject)"
    rec["gpu"], rec["power_limit"] = card()
    print(json.dumps(rec))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
