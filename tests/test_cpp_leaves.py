"""The leaf accessors of the C++ shim (tests/cpp/leaves_example.cpp) compile without PCL and link with libb200tsdf.so; on a
GPU box the example runs and its counts equal the Python mirror's on the same volume."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "leaves_example.cpp")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(engine_lib, out_dir):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(out_dir), "leaves_example")
    subprocess.run([CXX, "-std=c++17", "-O1", "-Wall", "-Werror", SRC, "-o", exe, f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}",
                    "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_leaf_accessors_compile_and_report_missing_device(engine_lib, tmp_path):
    exe = build(engine_lib, tmp_path)
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("device present: covered by the gpu test")
    except ImportError:
        pass
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr


@pytest.mark.gpu
def test_leaf_accessors_agree_with_the_python_mirror(engine_lib, tmp_path):
    import cpu_tsdf_b200 as pkg
    r = subprocess.run([build(engine_lib, tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    m = re.search(r"centers4=(\d+) centers-1=(\d+) occupied=(\d+) culled=(\d+) first_culled=(\S+)", r.stdout)
    assert m, r.stdout
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    v.setGridSize(3.0, 3.0, 3.0); v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, 319.5, 239.5)
    v.reset()
    u, w = np.meshgrid(np.arange(640, dtype=np.float32), np.arange(480, dtype=np.float32))
    cloud = np.zeros((480, 640, 4), np.float32)
    cloud[..., 0] = (u - np.float32(319.5)) / np.float32(525.0)
    cloud[..., 1] = (w - np.float32(239.5)) / np.float32(525.0)
    cloud[..., 2] = 1.0
    pose = np.eye(4); pose[2, 3] = -1.0
    for _ in range(3):
        v.integrateCloud(cloud, None, pose)
    mask = v.getFrustumCulledVoxels(pose)
    got = [int(m.group(i)) for i in range(1, 5)]
    assert got == [len(v.getVoxelCenters()), len(v.getVoxelCenters(-1)), len(v.getOccupiedVoxelIndices()), int(mask.sum())]
    # the first culled cell in depth-first order is the first set cell of the mask in bit-interleaved order
    c = v.getVoxelCenters(3)                      # the coarse cells (C = 3), depth first
    n = mask.shape[0]
    order = [(x, y, z) for x, y, z in (tuple(int(b) for b in np.floor((p + 1.5) / (3.0 / n))) for p in c)]
    first = next(i for i, (x, y, z) in enumerate(order) if mask[x, y, z])
    assert m.group(5) == ",".join(f"{a:.6f}" for a in c[first])
