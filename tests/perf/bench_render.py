#!/usr/bin/env python3
"""renderView speed after the 100-frame 2048^3 colour stream (the volume of tests/perf/bench_leaves.py), 640x480 views
along the orbit.  Reports, with the card's name and power limit read in the same run:

* renderViewBatchDevice for n = 1, 8 and 32 poses per call, plain and coloured: ms per view and rays per second (host clock
  around `repeats` calls that ends in a sync, so it covers the record upload and the launches);
* the single-pose renderView (image copied to the host and repacked into PointNormal), on this tree and, with --parent-lib,
  on another build of libb200tsdf.so, alternated round by round; the two must return the same bits;
* with --cpu, the reference's own renderView (oracle/_ref/libcpu_tsdf_ref.so, one core of the host) on the same volume.

    python tests/perf/bench_render.py [--parent-lib build/parent/libb200tsdf.so] [--cpu] [--out FILE]"""
import argparse
import ctypes as C
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

RES, SIZE = 2048, 10.0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:
        return None, None


def other_library(path):
    """another build of libb200tsdf.so, with the argument types of the entry points a volume needs to fuse and render"""
    lib, vp = C.CDLL(os.path.abspath(path)), C.c_void_p
    lib.b200tsdf_default_config.argtypes = [C.POINTER(pkg.Config)]
    lib.b200tsdf_create.argtypes = [C.POINTER(pkg.Config), C.POINTER(vp)]
    lib.b200tsdf_destroy.argtypes = [vp]
    lib.b200tsdf_last_error.argtypes = [vp]; lib.b200tsdf_last_error.restype = C.c_char_p
    lib.b200tsdf_set_config.argtypes = [vp, C.POINTER(pkg.Config)]
    lib.b200tsdf_reset.argtypes = [vp]
    lib.b200tsdf_integrate.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, vp]
    lib.b200tsdf_render.argtypes = [vp, vp, C.c_int, vp, C.c_size_t, C.c_int, C.c_int, vp]
    lib.b200tsdf_sync.argtypes = [vp]
    if hasattr(lib, "b200tsdf_render_batch_device"):
        lib.b200tsdf_render_batch_device.argtypes = [vp, C.c_int, vp, C.c_int, vp, C.c_size_t, C.c_int, C.c_int, vp]
    return lib


def volume(lib=None):
    if lib is None:
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=20)
    else:                                     # the Python mirror over another build of the library
        v = pkg.TSDFVolumeOctree.__new__(pkg.TSDFVolumeOctree)
        v._lib, v._cfg, v._h = lib, pkg.Config(), C.c_void_p()
        lib.b200tsdf_default_config(C.byref(v._cfg)); v._cfg.pool_log2 = 20
        assert lib.b200tsdf_create(C.byref(v._cfg), C.byref(v._h)) == 0
    cam = synth.Camera()
    v.setResolution(RES, RES, RES); v.setGridSize(SIZE, SIZE, SIZE)
    v.setCameraIntrinsics(525.0, 525.0, cam.cx, cam.cy); v.setIntegrateColor(True)
    v.reset()
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=8, help="calls per timed batch size")
    ap.add_argument("--rounds", type=int, default=5, help="alternated rounds of the single-pose comparison")
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    stream = list(frames(synth.S2, 100, stride=1, color=True, noise_seed=12345))
    v = volume()
    for pose, cloud in stream:
        v.integrateCloud(cloud, None, pose)
    v.sync()
    W, H = v._cfg.image_width, v._cfg.image_height
    views = [synth.orbit_pose(synth.S2, 3 * k + 1, 100) for k in range(32)]
    rec = {"what": "renderView after the 100-frame 2048^3 / 10 m colour stream, 640x480 views along the orbit",
           "batch_timing": f"host clock around {a.repeats} calls ending in a sync, after one warm-up call per shape"}
    out = torch.empty((32, H, W, 12), dtype=torch.float32, device="cuda")
    rgb = torch.empty((32, H, W, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def batch_seconds(vol, n, colored):
        call = lambda: vol.renderViewBatchDevice(views[:n], out.data_ptr(), d_rgb=rgb.data_ptr() if colored else None)
        call(); vol.sync()
        t0 = time.perf_counter()
        for _ in range(a.repeats):
            call()
        vol.sync()
        return (time.perf_counter() - t0) / (a.repeats * n)

    for colored in (False, True):
        for n in (1, 8, 32):
            s = batch_seconds(v, n, colored)
            key = f"batch{n}_{'colored' if colored else 'plain'}"
            rec[f"{key}_ms_per_view"] = round(s * 1e3, 3)
            rec[f"{key}_rays_per_s"] = round(W * H / s)
    # the batch's first image is the single-pose call's
    one = v.renderView(views[0])
    got = out[0].cpu().numpy()
    assert np.array_equal(got[..., :3].view(np.uint32), one[..., :3].view(np.uint32))
    rec["hit_pixels_view0"] = int(np.isfinite(one[..., 2]).sum())

    sides = {"this": v}
    if a.parent_lib:
        p = volume(other_library(a.parent_lib))
        for pose, cloud in stream:
            p.integrateCloud(cloud, None, pose)
        p.sync()
        sides["parent"] = p
        if hasattr(p._lib, "b200tsdf_render_batch_device"):          # both builds have the batch: time it alternately
            ts = {"this": [], "parent": []}
            for r in range(a.rounds):
                for name, vol in ((("this", v), ("parent", p)) if r % 2 == 0 else (("parent", p), ("this", v))):
                    ts[name].append(batch_seconds(vol, 32, False) * 1e3)
            for name, t in ts.items():
                rec[f"batch32_plain_{name}_alternated_ms_per_view"] = round(float(np.median(t)), 3)
    single = {k: [] for k in sides}
    first = {}
    for r in range(a.rounds):
        for name in (sides if r % 2 == 0 else list(sides)[::-1]):
            vol = sides[name]
            first.setdefault(name, vol.renderView(views[0]))          # warm-up, and the bits the sides must share
            t0 = time.perf_counter()
            for pose in views[:8]:
                vol.renderView(pose)
            single[name].append((time.perf_counter() - t0) / 8 * 1e3)
    for name, ts in single.items():
        rec[f"single_{name}_ms_per_view"] = round(float(np.median(ts)), 3)
        rec[f"single_{name}_ms_rounds"] = [round(t, 3) for t in ts]
    if "parent" in first:
        assert np.array_equal(np.nan_to_num(first["this"]).view(np.uint32), np.nan_to_num(first["parent"]).view(np.uint32))
        assert np.array_equal(np.isnan(first["this"]), np.isnan(first["parent"]))
        rec["single_timing"] = (f"renderView (copy to the host, repack), 8 views per round, {a.rounds} rounds alternating this "
                                "tree and the parent build, median")
    if a.cpu:
        from oracle.oracle_py import OracleVolume, REF_LIB
        if os.path.exists(REF_LIB):
            cam = synth.Camera()
            o = OracleVolume(kind="reference", xres=RES, yres=RES, zres=RES, xsize=SIZE, ysize=SIZE, zsize=SIZE,
                             integrate_color=1, cx=cam.cx, cy=cam.cy)
            o.reset()
            for pose, cloud in stream:
                o.integrate(cloud, pose)
            t0 = time.perf_counter()
            want = o.render(views[0])
            rec["cpu_reference_ms_per_view"] = round((time.perf_counter() - t0) * 1e3, 1)
            rec["cpu_reference"] = "the reference's own renderView on one host core, one view"
            assert np.array_equal(want[..., :3], one[..., :3], equal_nan=True)
    rec["gpu"], rec["power_limit"] = card()
    line = json.dumps(rec)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(rec, indent=1) + "\n")


if __name__ == "__main__":
    main()
