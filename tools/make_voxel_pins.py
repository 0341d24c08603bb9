#!/usr/bin/env python3
"""Generate tests/golden/voxel_pins.json from THE REFERENCE'S OWN METHODS: tsdf->octree_->getContainingVoxel (x, y, z,
min_size) and the returned node's getCenter / getSize / getData / getRGB / hasChildren, called on the reference build after
each case (oracle/_ref/libcpu_tsdf_ref_voxels.so, `make -f oracle/voxels.mk ref` where the reference tree exists), stored as
[count, SHA-256] of the records.  The point sets and min_size values are tests/voxels.py's; the dense crops are lookups at
getVoxelCenter over the boxes below.  tests/test_voxels.py replays them through the C++ restatement and the host emulation
(CPU), tests/test_voxels_gpu.py through the CUDA engine (GPU)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cpu_tsdf_b200 import synth  # noqa: E402
from tests import voxels  # noqa: E402
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, frames  # noqa: E402

CFG_512_12M = dict(xres=512, yres=512, zres=512, xsize=12.0, ysize=12.0, zsize=12.0, cx=CAM.cx, cy=CAM.cy,
                   max_cell_x=0.5, max_cell_y=0.5, max_cell_z=0.5)          # C = 5 > L - 6 = 3: two levels above C in the top brick
CFG_128 = dict(xres=128, yres=128, zres=128, xsize=3.0, ysize=3.0, zsize=3.0, cx=CAM.cx, cy=CAM.cy)
CFG_256_27 = dict(xres=256, yres=256, zres=256, xsize=2.7, ysize=2.7, zsize=2.7, cx=CAM.cx, cy=CAM.cy)

# name -> (config, scene, frames, stride, colour mode (None, "RGB", "RGBNormalized"), noise seed, dropout)
CASES = {
    "pin_256_5_9_rgb": (CFG_256, "S1", 5, 9, "RGB", 7, 0.01),
    "pin_256_3_9_rgbn": (CFG_256, "S1", 3, 9, "RGBNormalized", 7, 0.01),
    "pin_512_4_13_nocolor": (CFG_512, "S1", 4, 13, None, 7, 0.01),
    "pin_2048_2_3_rgb": (CFG_2048, "S2", 2, 3, "RGB", 7, 0.01),
    "shape_128_3m": (CFG_128, "S1", 2, 7, "RGB", 5, 0.0),
    "shape_256_2p7m": (CFG_256_27, "S1", 2, 7, None, 5, 0.0),
    "shape_512_12m": (CFG_512_12M, "shape", 2, 6, None, 9, 0.0),
    "empty_256": (CFG_256, "S1", 0, 1, "RGB", None, 0.0),
}
# finest-voxel boxes {i0, j0, k0, i1, j1, k1} per resolution: unaligned crops, a one-voxel slab and a box on the upper faces
BOXES = {
    128: [(40, 50, 60, 77, 70, 93), (0, 0, 0, 128, 128, 1), (100, 117, 120, 128, 128, 128)],
    256: [(90, 101, 77, 131, 140, 109), (3, 0, 250, 256, 256, 251), (230, 241, 200, 256, 256, 256)],
    512: [(200, 230, 190, 243, 262, 229), (255, 0, 0, 256, 512, 512), (480, 500, 497, 512, 512, 512)],
    2048: [(1000, 1010, 990, 1043, 1037, 1033), (1024, 900, 1000, 1025, 1100, 1100), (2030, 2040, 2001, 2048, 2048, 2048)],
}


def scene_of(name, cfg):
    if name == "shape":
        return synth.Scene(room_half=min(1.3, cfg["xsize"] * 0.45), cam_radius=0.8)
    return getattr(synth, name)


def color_kw(mode):
    return dict(integrate_color=int(mode is not None), color_mode=1 if mode == "RGBNormalized" else 0)


def stream(case):
    cfg, scene, n, stride, color, noise, dropout = case
    return frames(scene_of(scene, cfg), n, stride=stride, color=color is not None, noise_seed=noise, dropout=dropout)


def fuse(vol, case):
    for pose, cloud in stream(case):
        vol.integrate(cloud, pose)
    return vol


def oracle_volume(kind, case):
    """oracle `kind` ("port" = the C++ restatement, "reference" = oracle/_ref) with the point lookup, after the case's frames"""
    from oracle.voxels_py import VoxelsOracleVolume
    v = VoxelsOracleVolume(kind=kind, **color_kw(case[4]), **case[0])
    v.reset()
    return fuse(v, case)


def outputs(lookup, case):
    """name -> array: every point set at every min_size, then the dense crops of the case's resolution"""
    cfg = case[0]
    size, res = cfg["xsize"], cfg["xres"]
    finest = res.bit_length() - 1
    out = voxels.lookup_outputs(lookup, size, finest)
    for b in BOXES[res]:
        dense = voxels.dense_from_lookups(lambda p: lookup(p, -1.0), size, res, b)
        for k, a in dense.items():
            out[f"dense{list(b)}.{k}"] = a
    return out


def run_oracle(kind, case):
    v = oracle_volume(kind, case)
    return outputs(v.containing_voxels, case)


def digests(out):
    return {k: voxels.digest(a) for k, a in out.items()}


def main():
    from oracle import voxels_py
    if not os.path.exists(voxels_py.REF_LIB):
        raise SystemExit("oracle/_ref/libcpu_tsdf_ref_voxels.so is not built: run `make -f oracle/voxels.mk ref` where the reference tree exists")
    out = {"generator": "tools/make_voxel_pins.py",
           "source": "octree_->getContainingVoxel and the node accessors of oracle/_ref = the reference's src/lib/*.cpp compiled "
                     "verbatim (sdmiller/cpu_tsdf @ 9b973cb), called through oracle/ref_voxels_capi.cpp",
           "cases": {k: digests(run_oracle("reference", c)) for k, c in CASES.items()}}
    path = os.path.join(ROOT, "tests", "golden", "voxel_pins.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", path, {k: len(v) for k, v in out["cases"].items()})


if __name__ == "__main__":
    main()
