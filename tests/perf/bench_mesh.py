#!/usr/bin/env python3
"""Marching cubes and the mesh post-processing after the 100-frame 2048^3 / 10 m colour stream (the stream of bench.py and
tests/perf/bench_leaves.py), coloured by RGB at w_min 2.  Wall time on the host clock around calls that end synchronised; every
arm is called once to warm up, then the arms take turns for --repeats rounds and each reports its median:

* reconstruct() (the soup in host memory, copied into numpy arrays);
* reconstructDevice as a count query alone, as a count query followed by an emitting call, and as one emitting call with a
  known capacity (torch buffers);
* flattenVertices -> cleanupMesh on the host arrays, against flattenVerticesDevice (soup mode) -> cleanupMeshDevice on the
  device soup.

The device results are downloaded once and checked bit for bit against the host results.  With --profile, in a run of its own,
the device time of every kernel is taken from torch.profiler (CUDA activities) for one call of each of: the count query, the
emitting call with a known capacity (which walks the volume twice, counting and then emitting) and the device flatten ->
cleanup chain; it is added to the JSON written before under --out.  The card's name and power limit are read in the same run.

    python tests/perf/bench_mesh.py [--repeats 5] [--out profiles/h100_mesh.json]
    python tests/perf/bench_mesh.py --profile [--out profiles/h100_mesh.json]"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import cpu_tsdf_b200 as pkg  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402
from tests.common import frames  # noqa: E402

W_MIN, COLOR_MODE = 2.0, 1


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return None, None


def kernel_name(name):
    """the project's kernel (k_...<...>), the cub kernel's class, or the copy / memset as the profiler names it"""
    m = re.search(r"\b(k_\w+(?:<\w+>)?)", name)
    if m:
        return m.group(1)
    m = re.search(r"(Device\w+Kernel)", name)
    return "cub::" + m.group(1) if m else name.strip()


def interleaved(arms, repeats):
    """{name: fn} -> ({name: median ms}, {name: [ms per round]}, {name: last result}); one warm-up call each, then the arms take
    turns, so that a drift of the machine reaches all of them alike"""
    out = {k: fn() for k, fn in arms.items()}
    ts = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            t0 = time.perf_counter(); out[k] = fn(); ts[k].append((time.perf_counter() - t0) * 1e3)
    return {k: float(np.median(t)) for k, t in ts.items()}, ts, out


def volume():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, synth.Camera().cx, synth.Camera().cy); v.setIntegrateColor(True)
    v.reset()
    for pose, cloud in frames(synth.S2, 100, stride=1, color=True, noise_seed=12345):
        v.integrateCloud(cloud, None, pose)
    v.sync()
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(v); mc.setMinWeight(W_MIN); mc.setColorByRGB(COLOR_MODE == 1)
    return v, mc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--profile", action="store_true", help="per-kernel device times (torch.profiler), merged into --out")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_mesh.json"))
    a = ap.parse_args()
    import torch

    v, mc = volume()
    n = mc.reconstructDevice()
    d_v = torch.empty((n, 3), dtype=torch.float32, device="cuda"); d_c = torch.empty((n, 3), dtype=torch.uint8, device="cuda")
    f_v = torch.empty((n, 3), dtype=torch.float32, device="cuda"); f_t = torch.empty((n // 3, 3), dtype=torch.int32, device="cuda")
    c_v = torch.empty((n, 3), dtype=torch.float32, device="cuda"); c_t = torch.empty((n // 3, 3), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def count_query():
        return mc.reconstructDevice()

    def query_and_emit():
        m = mc.reconstructDevice()
        return mc.reconstructDevice(d_v.data_ptr(), m, d_c.data_ptr())

    def one_call():
        return mc.reconstructDevice(d_v.data_ptr(), n, d_c.data_ptr())

    def device_chain():
        nv, nt = pkg.flattenVerticesDevice(v, d_v.data_ptr(), n, None, n // 3, f_v.data_ptr(), f_t.data_ptr())
        return pkg.cleanupMeshDevice(v, f_v.data_ptr(), nv, f_t.data_ptr(), nt, c_v.data_ptr(), c_t.data_ptr())

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        one_call(); device_chain()                                        # warm-up outside the profiled window
        per = {}
        for arm, fn in (("reconstructDevice_count_query", count_query), ("reconstructDevice_known_capacity", one_call),
                        ("flatten_cleanup_device_soup", device_chain)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            ks = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    name = kernel_name(e.name)
                    ks[name] = ks.get(name, 0.0) + (getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0))
            per[arm] = {k: round(t / 1e3, 3) for k, t in sorted(ks.items(), key=lambda kv: -kv[1])}
        rec = {}
        if os.path.exists(a.out):
            with open(a.out) as f:
                rec = json.load(f)
        name, limit = card()
        rec["profile_ms_per_kernel"] = per
        rec["profile_ms_total"] = {arm: round(sum(ks.values()), 3) for arm, ks in per.items()}
        rec["profile_timing"] = ("torch.profiler (CUDA activities), device time summed per kernel name (ms) over one call of each arm, "
                                 "in a run of its own; reconstructDevice_known_capacity walks the volume twice (count, then emit)")
        rec["profile_gpu"], rec["profile_power_limit"] = name, limit
    else:
        verts, rgb, polys = mc.reconstruct()
        arms = {"reconstruct_host": mc.reconstruct, "reconstructDevice_count_query": count_query,
                "reconstructDevice_count_and_emit": query_and_emit, "reconstructDevice_known_capacity": one_call,
                "flatten_cleanup_host_arrays": lambda: pkg.cleanupMesh(*pkg.flattenVertices(verts, polys)),
                "flatten_cleanup_device_soup": device_chain}
        ms, rounds, out = interleaved(arms, a.repeats)
        assert out["reconstructDevice_count_query"] == out["reconstructDevice_count_and_emit"] == out["reconstructDevice_known_capacity"] \
            == n == len(verts)
        # the device soup equals the host soup bit for bit (the last call of the device arms wrote it)
        assert np.array_equal(d_v.cpu().numpy().view(np.uint32), verts.view(np.uint32)) and np.array_equal(d_c.cpu().numpy(), rgb)
        hv, ht = out["flatten_cleanup_host_arrays"]
        nv, nt = out["flatten_cleanup_device_soup"]
        assert np.array_equal(c_v[:nv].cpu().numpy().view(np.uint32), hv.view(np.uint32)) and np.array_equal(c_t[:nt].cpu().numpy(), ht)
        name, limit = card()
        rec = {"what": f"marching cubes (colour by RGB, w_min {W_MIN}) and flattenVertices -> cleanupMesh after the 100-frame "
                       "2048^3 / 10 m colour stream",
               "gpu": name, "power_limit": limit,
               "n_triangles": n // 3, "n_vertices_soup": n, "n_vertices_after_cleanup": int(nv), "n_triangles_after_cleanup": int(nt),
               "soup_bytes": n * 15,
               **{f"ms_{k}": round(t, 2) for k, t in ms.items()},
               "ms_per_round": {k: [round(x, 2) for x in t] for k, t in rounds.items()},
               "timing": f"host clock around calls that end synchronised; one warm-up call per arm, then {a.repeats} rounds in which "
                         "the arms take turns; median per arm",
               "checked": "device soup and device flatten -> cleanup downloaded and equal to the host results bit for bit",
               "reference_mesher": "not measured"}
    print(json.dumps(rec))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
