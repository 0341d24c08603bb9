#!/usr/bin/env python3
"""IncrementalMesh.update() against reconstructDevice with a known capacity, on a 2048^3 / 10 m colour volume coloured by RGB
at w_min 2.  Frames are fused in batches of 8 (integrateCloud, then sync, untimed); after each batch both arms mesh the volume,
in alternating order, each on the host clock around a call that ends synchronised.  The first two batches are warm-up; the
median over the remaining rounds is reported with the fraction of cells and of vertices each update re-meshed.  Every update
is checked bit for bit against the full mesh of the same round.  Two workloads:

* partial: the 100-frame orbit of bench.py first (untimed), then a slow sweep (an orbit of 800 frames, 8 per batch) in which
  each batch sees a part of the room: the case incremental meshing is for;
* orbit: bench.py's 100-frame orbit from an empty volume, where nearly every occupied cell is in view of every batch, so the
  helper can only add its own overhead.

The card's name and power limit are read in the same run.

    python tests/perf/bench_mesh_incremental.py [--rounds 10] [--out profiles/h100_mesh_incremental.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import cpu_tsdf_b200 as pkg  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402
from tests.common import frames  # noqa: E402
from tests.perf.bench_mesh import card  # noqa: E402

W_MIN, COLOR_MODE, BATCH = 2.0, 1, 8


def volume():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    v.setResolution(2048, 2048, 2048); v.setGridSize(10.0, 10.0, 10.0)
    v.setCameraIntrinsics(525.0, 525.0, synth.Camera().cx, synth.Camera().cy); v.setIntegrateColor(True)
    v.reset()
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(v); mc.setMinWeight(W_MIN); mc.setColorByRGB(COLOR_MODE == 1)
    return v, mc


def run(workload, rounds):
    import torch
    v, mc = volume()
    if workload == "partial":
        for pose, cloud in frames(synth.S2, 100, stride=1, color=True, noise_seed=12345):
            v.integrateCloud(cloud, None, pose)
        stream = list(frames(synth.S2, BATCH * (rounds + 2), stride=1, total=800, color=True, noise_seed=777))
    else:
        stream = list(frames(synth.S2, 100, stride=1, color=True, noise_seed=12345))
    inc = pkg.IncrementalMesh(v, W_MIN, COLOR_MODE)
    inc.update()
    cap = 0
    d_v = d_c = None
    t_inc, t_full, frac_cells, frac_verts, sizes = [], [], [], [], []
    nbatches = len(stream) // BATCH
    for b in range(nbatches):
        for pose, cloud in stream[b * BATCH:(b + 1) * BATCH]:
            v.integrateCloud(cloud, None, pose)
        v.sync()
        n = mc.reconstructDevice()                       # the known capacity of the full arm (untimed)
        if n > cap:
            cap = n + n // 4
            d_v = torch.empty((cap, 3), dtype=torch.float32, device="cuda"); d_c = torch.empty((cap, 3), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()

        def full():
            t0 = time.perf_counter(); m = mc.reconstructDevice(d_v.data_ptr(), cap, d_c.data_ptr()); return m, (time.perf_counter() - t0) * 1e3

        def incremental():
            t0 = time.perf_counter(); out = inc.update(); torch.cuda.synchronize(); return out, (time.perf_counter() - t0) * 1e3

        if b % 2:
            (m, tf), ((iv, ic), ti) = full(), incremental()
        else:
            ((iv, ic), ti), (m, tf) = incremental(), full()
        assert m == n == iv.shape[0]
        assert torch.equal(iv.view(torch.int32), d_v[:n].view(torch.int32)) and torch.equal(ic, d_c[:n]), "update differs from the full mesh"
        if b < 2:
            continue
        ncells = v.changedCells(0)[1].size
        t_inc.append(ti); t_full.append(tf)
        frac_cells.append(inc.cells_remeshed / ncells); frac_verts.append(inc.verts_remeshed / max(n, 1)); sizes.append(n)
    med = lambda x: float(np.median(x))
    return {"rounds": len(t_inc), "frames_per_update": BATCH,
            "update_ms_median": med(t_inc), "reconstructDevice_known_capacity_ms_median": med(t_full),
            "speedup_median": med(t_full) / med(t_inc),
            "update_ms": [round(t, 3) for t in t_inc], "reconstructDevice_ms": [round(t, 3) for t in t_full],
            "cells_remeshed_fraction_median": med(frac_cells), "verts_remeshed_fraction_median": med(frac_verts),
            "mesh_vertices_median": int(med(sizes))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=10, help="timed rounds per workload (two more are warm-up)")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_mesh_incremental.json"))
    a = ap.parse_args()
    name, limit = card()
    res = {"card": name, "power_limit": limit, "grid": "2048^3 / 10 m, colour, w_min 2, RGB",
           "partial": run("partial", a.rounds), "orbit": run("orbit", a.rounds)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
