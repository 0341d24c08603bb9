"""getContainingVoxel of the C++ shim (tests/cpp/voxels_example.cpp) compiles without PCL and links with libb200tsdf.so; on a
GPU box the example runs and its records equal the Python mirror's on the same volume."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "voxels_example.cpp")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(engine_lib, out_dir):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(out_dir), "voxels_example")
    subprocess.run([CXX, "-std=c++17", "-O1", "-Wall", "-Werror", SRC, "-o", exe, f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}",
                    "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_voxel_lookup_compiles_and_reports_missing_device(engine_lib, tmp_path):
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
def test_voxel_lookup_agrees_with_the_python_mirror(engine_lib, tmp_path):
    import cpu_tsdf_b200 as pkg
    r = subprocess.run([build(engine_lib, tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    v.setGridSize(3.0, 3.0, 3.0); v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, 319.5, 239.5)
    v.setIntegrateColor(True)
    v.reset()
    u, w = np.meshgrid(np.arange(640, dtype=np.float32), np.arange(480, dtype=np.float32))
    cloud = np.zeros((480, 640, 8), np.float32)
    cloud[..., 0] = (u - np.float32(319.5)) / np.float32(525.0)
    cloud[..., 1] = (w - np.float32(239.5)) / np.float32(525.0)
    cloud[..., 2] = 1.0
    cloud.view(np.uint8).reshape(480, 640, 32)[..., 16:20] = (50, 100, 200, 255)     # b, g, r, a
    pose = np.eye(4); pose[2, 3] = -1.0
    for _ in range(3):
        v.integrateCloud(cloud, None, pose)
    pts = np.array([[0.01, 0.02, 0.003], [0.01, 0.02, 0.003], [2.0, 0.0, 0.0], [0.3, -0.2, 0.9]], np.float32)
    lines = re.findall(r"voxel \d: (.*)", r.stdout)
    assert len(lines) == 4, r.stdout
    for i, (p, ms) in enumerate(zip(pts, (-1.0, 0.1, -1.0, -1.0))):
        rec = v.getContainingVoxels(p[None], ms)[0]
        valid = rec["level"] >= 0
        c = [rec["cx"], rec["cy"], rec["cz"]] if valid else [0.0] * 3
        want = (f"valid={int(valid)} depth={rec['level']} d={float(rec['d']) if valid else 0:.9g} w={float(rec['w']) if valid else 0:.9g} "
                f"c={float(c[0]):.9g},{float(c[1]):.9g},{float(c[2]):.9g} size={float(rec['size']) if valid else 0:.9g} "
                f"rgb={rec['r']},{rec['g']},{rec['b']} children={rec['has_children']}")
        assert lines[i] == want, (i, lines[i], want)
    assert "valid=0" in lines[2] and "children=1" in lines[1] and "w=0 " not in lines[0]
