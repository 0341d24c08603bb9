"""trackDepthImage of the C++ shim (tests/cpp/track_example.cpp) compiles without PCL and links with libb200tsdf.so; on a GPU
box the example runs and prints what the Python mirror gives for the same calls on the same volume."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "track_example.cpp")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(engine_lib, out_dir):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(out_dir), "track_example")
    subprocess.run([CXX, "-std=c++17", "-O1", "-Wall", "-Werror", SRC, "-o", exe, f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}",
                    "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_tracking_compiles_and_reports_missing_device(engine_lib, tmp_path):
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
def test_tracking_agrees_with_the_python_mirror(engine_lib, tmp_path):
    import cpu_tsdf_b200 as pkg
    r = subprocess.run([build(engine_lib, tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=14)
    v.setGridSize(3.0, 3.0, 3.0); v.setResolution(256, 256, 256); v.setCameraIntrinsics(525.0, 525.0, 319.5, 239.5)
    v.reset()
    W, H = 640, 480
    u, w = np.meshgrid(np.arange(W), np.arange(H))
    d16 = (1000 + u // 8 + w // 16).astype(np.uint16)
    d32 = d16.astype(np.float32) * np.float32(1e-3)
    pose = np.eye(4); pose[2, 3] = -1.0
    for _ in range(2):
        v.integrateDepth(d16, pose, None, 1e-3)
    a = pose.copy(); a[0, 3] = 0.01
    pa, ra = v.trackDepth(d16, a, None, 1e-3)
    b = pose.copy(); b[2, 3] = -1.02
    pb, _ = v.trackDepth(d32, b, None, 1.0)
    with pytest.raises(pkg.B200Error):
        v.trackDepth(d32, b, pkg.TrackParams.default(levels=0), 1.0)
    want = [f"u16: {ra['status']} {ra['inliers']} {pa[0, 3]:.17g} {pa[1, 3]:.17g} {pa[2, 3]:.17g}",
            f"f32: {pb[0, 3]:.17g} {pb[1, 3]:.17g} {pb[2, 3]:.17g}", "refused: 1 -1"]
    assert r.stdout.strip().splitlines() == want
    assert abs(pb[2, 3] + 1.0) < abs(b[2, 3] + 1.0)                      # a wall pins the depth direction
