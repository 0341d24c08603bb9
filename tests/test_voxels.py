"""getContainingVoxel and the dense crop without a GPU.

tests/golden/voxel_pins.json holds digests of what the reference's own octree_->getContainingVoxel and node accessors return
on the reference build (tools/make_voxel_pins.py, oracle/ref_voxels_capi.cpp): point sets (uniform, on splitting planes, on
and one ulp outside the faces, NaN, -0.0) at a sweep of min_size, and dense crops as lookups at getVoxelCenter.  The C++
restatement (oracle/tsdf_oracle_voxels.cpp) must reproduce them, and equal the reference's live records where oracle/_ref is
built.  The host emulation of k_voxels and k_dense (tests/emu/voxels_emu.cpp: the kernels' own routines over the flat layout)
must equal the restatement field for field.  k_dense descends by index where the contract is the float descent at the voxel
centre; the two agree axis by axis, which is checked here for every voxel index on every grid shape the tests use."""
import importlib.util
import json
import os
import subprocess

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from oracle import voxels_py
from tests import voxels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("make_voxel_pins", os.path.join(ROOT, "tools", "make_voxel_pins.py"))
mvp = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mvp)
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "voxel_pins.json")))

# (resolution, size) of every volume the voxel tests fuse, on the CPU or the GPU
SHAPES = [(128, 3.0), (1024, 3.0), (256, 2.7), (512, 12.0), (256, 3.0), (512, 3.0), (2048, 10.0), (4096, 10.0)]


def assert_same(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("name", sorted(mvp.CASES))
def test_restatement_reproduces_reference_lookups(name):
    case = mvp.CASES[name]
    port = mvp.run_oracle("port", case)
    assert mvp.digests(port) == PINS["cases"][name]
    if os.path.exists(voxels_py.REF_LIB):
        assert_same(mvp.run_oracle("reference", case), port)             # the reference's own methods, live


def test_pins_are_not_trivial():
    case = mvp.CASES["pin_256_5_9_rgb"]
    out = mvp.run_oracle("port", case)
    faces = out["faces@-1.0"]
    assert (faces["level"] == -1).sum() == 20 and (faces["level"] >= 0).sum() == 20       # the ulp-outside points only
    sp = out["special@-1.0"]
    assert sp["level"][0] == -1 and (sp["level"][1:] >= 0).all()                          # NaN z is NULL, NaN x / y are not
    assert (out["uniform@-1.0"]["w"] > 0).sum() > 0 and (out["uniform@-1.0"]["r"] > 0).any()
    assert (out["uniform@0.375"]["has_children"] == 1).any()                               # stopped above a leaf
    u = out["uniform@4.5"]["level"]
    assert (u == 0).sum() > 3000 and (u <= 0).all()                                         # min_size above the root size
    d = out["dense[90, 101, 77, 131, 140, 109].w"]
    assert (d > 0).any() and (d == 0).any()
    nc = mvp.run_oracle("port", mvp.CASES["pin_512_4_13_nocolor"])["uniform@-1.0"]
    assert (nc["r"][nc["level"] >= 0] == 127).all()


def _emu(case):
    from tests.emu.voxels_py import EmuVoxelsVolume
    cfg = case[0]
    e = EmuVoxelsVolume(pool_log2=18 if cfg["xres"] >= 2048 else 16, **mvp.color_kw(case[4]), **cfg)
    e.reset()
    return mvp.fuse(e, case)


# the host emulation carries no RGBNormalized payload; that case runs on the GPU (tests/test_voxels_gpu.py)
@pytest.mark.parametrize("name", sorted(k for k, c in mvp.CASES.items() if c[4] != "RGBNormalized"))
def test_emulated_kernels_equal_the_restatement(name):
    case = mvp.CASES[name]
    cfg = case[0]
    want = mvp.run_oracle("port", case)
    e = _emu(case)
    got = mvp.outputs(e.containing_voxels, case)                       # k_voxels' routine (find_voxel)
    assert_same(got, want)
    for b in mvp.BOXES[cfg["xres"]]:                                    # k_dense's per-tile walk and per-voxel resolution
        dense = e.dense(b)
        for k, a in dense.items():
            assert a.tobytes() == want[f"dense{list(b)}.{k}"].tobytes(), (name, b, k)


@pytest.mark.parametrize("res,size", SHAPES)
def test_index_descent_equals_float_descent_per_axis(res, size):
    """k_dense takes the child bit of voxel i at level l as bit (L-1-l) of i; the contract is (v_i - ctr) > 0 in float at the
    voxel centre v_i.  The child choice on each axis depends only on that coordinate, so checking every i < res on each axis
    covers every voxel of the grid: 3 * res descents."""
    L = res.bit_length() - 1
    i = np.arange(res)
    want = ((i[None, :] >> (L - 1 - np.arange(L))[:, None]) & 1).astype(np.uint8)
    for _axis in range(3):                                              # cubic grids: the three axes share size and resolution
        v = voxels.voxel_centers_1d(size, res, i)
        assert np.array_equal(voxels.float_descent_bits(size, L, v), want)


def test_ctypes_voxel_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200tsdf.h"\nint main (void) {\n'
                   '  printf ("%zu", sizeof (b200tsdf_voxel));\n'
                   + "".join(f'  printf (" %zu", offsetof (b200tsdf_voxel, {f}));\n' for f, _ in pkg.Voxel._fields_)
                   + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    import ctypes
    assert got[0] == 44 == ctypes.sizeof(pkg.Voxel) == pkg.VOXEL_DTYPE.itemsize == voxels_py.VOXEL_DTYPE.itemsize
    assert got[1:] == [getattr(pkg.Voxel, f).offset for f, _ in pkg.Voxel._fields_]
    assert got[1:] == [pkg.VOXEL_DTYPE.fields[f][1] for f, _ in pkg.Voxel._fields_]
    assert pkg.VOXEL_DTYPE == voxels_py.VOXEL_DTYPE
