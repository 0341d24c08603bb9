"""integrateDepthImage of the C++ shim (tests/cpp/depth_example.cpp) compiles without PCL and links with libb200tsdf.so; on a
GPU box the example runs and prints what the Python mirror gives for the same calls on the same volume."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "depth_example.cpp")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(engine_lib, out_dir):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(out_dir), "depth_example")
    subprocess.run([CXX, "-std=c++17", "-O1", "-Wall", "-Werror", SRC, "-o", exe, f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}",
                    "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_depth_images_compile_and_report_missing_device(engine_lib, tmp_path):
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
def test_depth_images_agree_with_the_python_mirror(engine_lib, tmp_path):
    import cpu_tsdf_b200 as pkg
    r = subprocess.run([build(engine_lib, tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    v.setGridSize(3.0, 3.0, 3.0); v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, 319.5, 239.5)
    v.setIntegrateColor(True)
    v.reset()
    W, H = 640, 480
    u, w = np.meshgrid(np.arange(W), np.arange(H))
    hole = (u > 300) & (u < 340) & (w > 220) & (w < 260)
    d16 = np.where(hole, 0, 1000 + u // 8).astype(np.uint16)
    d32 = np.where(hole, np.float32(0), np.float32(1.0) + np.float32(0.0005) * w.astype(np.float32)).astype(np.float32)
    rgb = np.stack([u // 3, w // 2, np.full_like(u, 77)], axis=-1).astype(np.uint8)
    pose = np.eye(4); pose[2, 3] = -1.0
    for _ in range(2):
        v.integrateDepth(d16, pose, rgb, 1e-3)
    v.integrateDepth(d32, pose, None, 1.0)
    with pytest.raises(pkg.B200Error):
        v.integrateDepth(d16, pose, None, 0.0)
    pts = np.array([[0.0, 0.0, 0.0], [0.1, -0.05, 0.02], [-0.3, 0.2, -0.01], [0.0, 0.0, 0.5]], np.float32)
    ok, val = v.getFxn(pts)
    want = ["refused: 1 -1"] + [f"fxn {i}: {int(ok[i])} {float(val[i]) if ok[i] else 0.0:.9g}" for i in range(4)]
    assert r.stdout.strip().splitlines() == want
    assert ok.any()
