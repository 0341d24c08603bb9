"""Batched organise of unorganised clouds, without a GPU: the per-point mapping of k_org_zmin (flat index of the batch's
concatenated points -> frame and index within the frame, key, tie rule) compiled for the host (tests/emu/org_batch_emu.cpp) and
driven over frames of unequal size against the restatement of the reference's `integrate` program (oracle/prog_oracle.cpp);
and the ctypes signature of b200tsdf_integrate_unorganized_batch_device against include/b200tsdf.h."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from cpu_tsdf_b200 import synth
from oracle import oracle_py
from tests.common import CAM
from tests.test_organize import INTR, same_cloud, unorganized_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
vp = C.c_void_p


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("orgemu") / "liborgbatch.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++",
                    os.path.join(ROOT, "tests", "emu", "org_batch_emu.cpp"), "-o", lib], check=True)
    so = C.CDLL(lib)
    so.emu_organize_batch.argtypes = [C.c_int, vp, vp, C.c_size_t, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_float, C.c_int, vp,
                                      vp, C.c_size_t, C.c_int, vp, vp, vp]
    return so


def organize_batch(emu, clouds, *, rgba_off=16, cloud_units=1.0, zero_nans=False, worlds_to_camera=None):
    W, H = CAM.width, CAM.height
    m = len(clouds)
    ptrs = (vp * m)(*[c.ctypes.data if len(c) else None for c in clouds])
    counts = np.array([len(c) for c in clouds], np.uint64)
    strides = {c.shape[1] * 4 for c in clouds}
    assert len(strides) == 1
    tf = None if worlds_to_camera is None else np.ascontiguousarray(np.stack(worlds_to_camera), np.float64)
    out = np.full((m, H, W, 8), 7.0, np.float32)                       # pre-filled: padding must come back zero
    zkey = np.zeros(m * H * W, np.uint64); filled = np.zeros(m, np.int64)
    total = int(counts.sum()); fmap = np.zeros((max(total, 1), 2), np.uint64)
    intr = np.asarray(INTR, np.float32)
    rc = emu.emu_organize_batch(m, ptrs, counts.ctypes.data, strides.pop(), 0, rgba_off, intr.ctypes.data, W, H, float(cloud_units),
                                int(zero_nans), None if tf is None else tf.ctypes.data, out.ctypes.data, 32, 16, zkey.ctypes.data,
                                filled.ctypes.data, fmap.ctypes.data)
    assert rc == 0
    return out, zkey.reshape(m, H * W), filled, fmap[:total]


def test_flat_index_maps_to_frame_and_local_index(emu):
    """Frames of unequal size, empty ones at the start, in the middle and at the end: every flat index lands in its own frame at
    its own index, and each image is the restatement's organisation of that frame alone (duplicates: the earliest point wins)."""
    rng = np.random.default_rng(5)
    clouds = []
    for i, n in enumerate([0, 70000, 1, 0, 25000, 120000, 0]):
        pts, _ = unorganized_cloud(20 + i)
        clouds.append(np.ascontiguousarray(pts[:n]) if n else np.zeros((0, 8), np.float32))
    clouds[2] = clouds[5][rng.integers(0, 1000, 1)].copy()
    out, zkey, filled, fmap = organize_batch(emu, clouds)
    counts = [len(c) for c in clouds]
    want_f = np.repeat(np.arange(len(clouds)), counts)
    want_j = np.concatenate([np.arange(n) for n in counts])
    assert np.array_equal(fmap[:, 0], want_f) and np.array_equal(fmap[:, 1], want_j)
    for f, c in enumerate(clouds):
        want, nf = oracle_py.organize(c, INTR, CAM.width, CAM.height, rgba_off=16)
        assert filled[f] == nf and same_cloud(want, out[f]), f
        # key = z bits << 32 | index within the frame, and that index names a point with the winning z
        win = zkey[f] != np.uint64(~np.uint64(0))
        assert win.sum() == nf
        j = (zkey[f][win] & np.uint64(0xffffffff)).astype(np.int64)
        zb = (zkey[f][win] >> np.uint64(32)).astype(np.uint32)
        assert (j < len(c)).all()
        assert np.array_equal(c[j, 2].view(np.uint32), zb)
        assert np.array_equal(want.reshape(-1, 8)[win, 2].view(np.uint32), zb)


def test_ties_go_to_the_earliest_point_of_the_frame(emu):
    """Exact duplicates of one point at different flat positions: the winner's key holds the smallest index within its frame, not
    the smallest flat index, and a duplicate in another frame does not compete."""
    p = np.zeros((1, 8), np.float32); p[0, :3] = (0.0, 0.0, 1.5)                     # on the optical axis: every z hits the same pixel
    p[0, 4] = np.array([1, 2, 3, 4], np.uint8).view(np.float32)[0]
    q = p.copy(); q[0, 4] = np.array([9, 9, 9, 9], np.uint8).view(np.float32)[0]
    far = p.copy(); far[0, 2] = 2.0
    a = np.concatenate([far, q, p, q])                                  # frame 0: index 1 (q) wins the tie with 2 and 3
    b = np.concatenate([p, q])                                          # frame 1: index 0 (p) wins
    out, zkey, filled, _ = organize_batch(emu, [a, b])
    assert (filled == [1, 1]).all()
    k0 = zkey[0][zkey[0] != np.uint64(~np.uint64(0))]; k1 = zkey[1][zkey[1] != np.uint64(~np.uint64(0))]
    assert int(k0[0]) & 0xffffffff == 1 and int(k1[0]) & 0xffffffff == 0
    for f, c in enumerate((a, b)):
        want, _ = oracle_py.organize(c, INTR, CAM.width, CAM.height, rgba_off=16)
        assert same_cloud(want, out[f])


def test_per_frame_world_transform_units_and_zero_nans(emu):
    clouds, w2cs = [], []
    for i, n in enumerate([40000, 90000, 15000]):
        world = synth.orbit_pose(synth.S1, 7 + 11 * i, 100)
        pts, _ = unorganized_cloud(40 + i, scale=0.001, world_pose=world)
        clouds.append(np.ascontiguousarray(pts[:n])); w2cs.append(np.linalg.inv(world))
    kw = dict(cloud_units=0.001, zero_nans=True)
    out, _, filled, _ = organize_batch(emu, clouds, worlds_to_camera=w2cs, **kw)
    for f, c in enumerate(clouds):
        want, nf = oracle_py.organize(c, INTR, CAM.width, CAM.height, rgba_off=16, world_to_camera=w2cs[f], **kw)
        assert filled[f] == nf and nf > 1000 and same_cloud(want, out[f]), f


def _header_params(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200tsdf.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", src)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def _ctype_of(decl):
    t = re.sub(r"\s*\b\w+$", "", decl)                                 # drop the parameter name
    if "*" in t:
        return "ptr:" + re.sub(r"\bconst\b|\*|\s", "", t)
    return {"int": "int", "size_t": "size_t"}[t]


def test_ctypes_signature_matches_the_header(engine_lib):
    import cpu_tsdf_b200 as pkg
    name = "b200tsdf_integrate_unorganized_batch_device"
    lib = pkg.load_library()
    assert name in pkg.EXPORTS
    want = [_ctype_of(p) for p in _header_params(name)]
    assert want == ["ptr:b200tsdf_t", "int", "ptr:void", "ptr:size_t", "size_t", "int", "int", "ptr:b200tsdf_organize_opts", "ptr:double"]
    got = getattr(lib, name).argtypes
    assert len(got) == len(want)
    for w, g in zip(want, got):
        if w == "int":
            assert g is C.c_int
        elif w == "size_t":
            assert g is C.c_size_t
        elif w == "ptr:size_t":
            assert g is C.POINTER(C.c_size_t)
        elif w == "ptr:b200tsdf_organize_opts":
            assert g is C.POINTER(pkg.OrganizeOpts)
        else:
            assert g is C.c_void_p, (w, g)
    assert getattr(lib, name).restype is C.c_int
