"""The C++ shim (include/cpu_tsdf_b200/tsdf_volume_octree.h) compiles against the C ABI and links
with libb200tsdf.so; on a GPU box the README-style example also runs end to end."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "shim_example.cpp")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(engine_lib, out_dir):
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(out_dir), "shim_example")
    subprocess.run([CXX, "-std=c++17", "-O1", SRC, "-o", exe, f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}",
                    "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    return exe


def test_shim_compiles_and_reports_missing_device(engine_lib, tmp_path):
    exe = build(engine_lib, tmp_path)
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("device present: covered by the gpu test")
    except ImportError:
        pass
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 3, r.stdout + r.stderr          # B200TSDF_ENODEVICE surfaced, no CPU fallback


@pytest.mark.gpu
def test_shim_example_runs(engine_lib, tmp_path):
    exe = build(engine_lib, tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "mesh:" in r.stdout


def test_host_packing_is_bit_preserving_and_the_pool_runs_every_job_once(tmp_path):
    """cpu_tsdf_b200/csrc/host_pack.h (the host half of the batched upload): tests/cpp/pack_test.cpp checks the packed pixels
    against the source bytes for the SSE and the generic paths, and the fork/join pool under run() and begin()/help()/end()."""
    exe = str(tmp_path / "pack_test")
    subprocess.run([CXX, "-std=c++17", "-O2", "-pthread", os.path.join(ROOT, "tests", "cpp", "pack_test.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "OK", r.stdout + r.stderr
