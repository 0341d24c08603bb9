#!/usr/bin/env python3
""".vol save and load after the 100-frame 2048^3 / 10 m colour stream: the device writer and parser (DESIGN.md §3e) against
the host writer and loader (debug_flags bit 2) on one build, alternating the two in every round.  Records the median and
range of the wall time of save, load, saveDevice and loadDevice, the CUDA-event time of the device-image calls, the file
size, and load followed by marching cubes (what b200_tsdf2mesh does after its argument parsing).  Files go to a temporary
directory; its file system is named in the record.  Prints one JSON line and writes it to --out.

    python tests/perf/bench_vol_io.py [--rounds 5] [--out profiles/h100_vol_io.json]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import cpu_tsdf_b200 as pkg  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402
from tests.common import frames  # noqa: E402

HOST_IO = 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return [s.strip() for s in q.split(",")]
    except Exception:
        return [None, None]


def fs_of(path):
    try:
        return subprocess.run(["stat", "-f", "-c", "%T", path], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        return None


def flags(v, f):
    v._cfg.debug_flags = f
    v._push()


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter(); fn(); t1 = time.perf_counter()
    return (t1 - t0) * 1e3


def events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter(); a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b), (time.perf_counter() - t0) * 1e3


def stat(xs):
    return {"median": round(float(np.median(xs)), 2), "min": round(float(np.min(xs)), 2), "max": round(float(np.max(xs)), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    cam = synth.Camera()
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, cam.cx, cam.cy); v.setIntegrateColor(True)
    v.reset()
    for pose, cloud in frames(synth.S2, 100, stride=1, color=True, noise_seed=12345):
        v.integrateCloud(cloud, None, pose)
    v.sync()
    tmp = tempfile.mkdtemp(prefix="vol_io_")
    try:
        paths = {m: os.path.join(tmp, f"{m}.vol") for m in ("device", "host")}
        w = {m: pkg.TSDFVolumeOctree(device=0, pool_log2=20) for m in paths}
        for m, f in (("device", 0), ("host", HOST_IO)):
            flags(w[m], f)
        t = {k: [] for k in ("save_device", "save_host", "load_device", "load_host", "load_mesh_device", "load_mesh_host",
                             "saveDevice_wall", "saveDevice_events", "loadDevice_wall", "loadDevice_events")}
        n = v.saveDevice()
        buf = torch.empty(n, dtype=torch.uint8, device="cuda")
        mc = pkg.MarchingCubesTSDFOctree(); mc.setMinWeight(2.0)
        for r in range(a.rounds + 1):                 # round 0 warms every path up and is not recorded
            order = ("device", "host") if r % 2 == 0 else ("host", "device")
            rec = {}
            for m in order:
                flags(v, 0 if m == "device" else HOST_IO)
                rec[f"save_{m}"] = wall(lambda: v.save(paths[m]))
            flags(v, 0)
            for m in order:
                rec[f"load_{m}"] = wall(lambda: w[m].load(paths[m]))
            for m in order:
                def load_mesh():
                    w[m].load(paths[m]); mc.setInputTSDF(w[m]); mc.reconstruct()
                rec[f"load_mesh_{m}"] = wall(load_mesh)
            rec["saveDevice_events"], rec["saveDevice_wall"] = events(lambda: v.saveDevice(buf.data_ptr(), n))
            rec["loadDevice_events"], rec["loadDevice_wall"] = events(lambda: w["device"].loadDevice(buf.data_ptr(), n))
            if r:
                for k, x in rec.items():
                    t[k].append(x)
        same = open(paths["device"], "rb").read() == open(paths["host"], "rb").read() == buf.cpu().numpy().tobytes()
        name, limit = card()
        out = {"what": ".vol save / load after the 100-frame 2048^3 / 10 m colour stream", "gpu": name, "power_limit": limit,
               "host_cpu": os.uname().machine, "file_system": fs_of(tmp), "file_bytes": os.path.getsize(paths["device"]),
               "n_leaves": int(len(v.getVoxelCenters(-1))), "bytes_identical": bool(same),
               "timing": f"ms, median and range of {a.rounds} rounds, device and host paths alternating; wall = host clock "
                         "around the synchronous call, events = CUDA events around it",
               **{k: stat(x) for k, x in t.items()}}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
