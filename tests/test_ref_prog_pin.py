"""Pins oracle/prog_oracle.cpp (the restatement of the reference's program-side functions) to the reference's OWN text of
src/prog/integrate.cpp, compiled from the source where it lies (oracle/Makefile `refprog`: meshToFaceCloud, flattenVertices,
cleanupMesh, reprojectPoint, lines 63-222; the per-cloud preparation + z-buffer re-organisation of main(), lines 559-635).
The restatement's outputs must reproduce the digests of that build's outputs stored in tests/golden/ref_pins.json
(tools/make_ref_pins.py); where oracle/_ref/libcpu_tsdf_refprog.so is built, its live outputs must reproduce them as well."""
import json
import os

import numpy as np
import pytest

from oracle import oracle_py
from tests.common import digests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_pins.json")))["ref_prog_pin"]


def pinned(key, run):
    """run("port") must reproduce the stored digests of run("reference"); returns the port's outputs"""
    got = run("port")
    assert digests(got) == PINS[key]
    if os.path.exists(oracle_py.REFPROG_LIB):
        assert digests(run("reference")) == PINS[key]
    return got


def _cloud(rng, n, spread=1.0):
    z = rng.uniform(0.4, 3.0, n).astype(np.float32)
    x = (rng.uniform(-0.7, 0.7, n) * z * spread).astype(np.float32)
    y = (rng.uniform(-0.55, 0.55, n) * z * spread).astype(np.float32)
    pts = np.zeros((n, 8), np.float32)
    pts[:, 0], pts[:, 1], pts[:, 2], pts[:, 3] = x, y, z, 1.0
    pts.view(np.uint32)[:, 4] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    return pts


@pytest.mark.parametrize("seed,units,zero_nans,world", [(1, 1.0, False, False), (2, 0.001, True, False), (3, 1.0, True, True), (4, 2.5, False, True)])
def test_organise_block_matches_the_reference_text(seed, units, zero_nans, world):
    rng = np.random.default_rng(seed)
    W, H = 160, 120
    intr = (131.25, 131.25, 79.5, 59.5)
    pts = _cloud(rng, 60000, spread=1.2)
    pts[:, :3] /= units                                            # the program scales by cloud_units first (:559-568)
    pts[rng.random(len(pts)) < 0.03, :3] = 0.0                     # (0,0,0) = NaN under --zero-nans
    pts[rng.random(len(pts)) < 0.02, 2] = np.nan
    pts[rng.random(len(pts)) < 0.02, 2] *= -1                      # behind the camera
    dup = rng.integers(0, len(pts), 4000)                          # exact depth ties: the earlier point must win (:603-606)
    pts[dup[:2000]] = pts[dup[2000:]]
    tf = None
    if world:
        a = 0.3 * seed
        tf = np.array([[np.cos(a), 0, np.sin(a), 0.1], [0, 1, 0, -0.05], [-np.sin(a), 0, np.cos(a), 0.2], [0, 0, 0, 1]], np.float64)
    kw = dict(rgba_off=16, cloud_units=units, zero_nans=zero_nans, world_to_camera=tf)

    def run(kind):
        a, na = oracle_py.organize(pts, intr, W, H, kind=kind, **kw)
        # x, y, z and the colour word; the padding float and the bytes after the colour are whatever the default point holds
        return {"filled": na, "xyz": a.view(np.uint32)[..., :3], "bgra": a.view(np.uint32)[..., 4]}
    assert pinned(f"organise_{seed}", run)["filled"] > 500


def _mc_like_mesh(rng, n_quads, jitter):
    """A bumpy sheet of quads split into triangles, as a soup (every triangle has its own three vertices, like marching cubes
    output), plus a few small stray islands for cleanupMesh."""
    g = int(np.sqrt(n_quads))
    xs, ys = np.meshgrid(np.arange(g + 1), np.arange(g + 1), indexing="ij")
    P = np.stack([xs * 0.01, ys * 0.01, 0.02 * np.sin(xs * 0.3) * np.cos(ys * 0.2)], -1).astype(np.float32)
    tris = []
    for i in range(g):
        for j in range(g):
            a, b, c, d = P[i, j], P[i + 1, j], P[i + 1, j + 1], P[i, j + 1]
            tris += [(a, b, c), (a, c, d)]
    for k in range(12):                                            # islands of 1..6 triangles far from the sheet
        o = np.array([0.5 + 0.2 * k, 1.0, 0.3], np.float32)
        for t in range(1 + k % 6):
            tris.append((o + [0.004 * t, 0, 0], o + [0.004 * t + 0.003, 0, 0], o + [0.004 * t, 0.003, 0]))
    soup = np.asarray(tris, np.float32).reshape(-1, 3)
    soup = soup + (rng.normal(scale=jitter, size=soup.shape)).astype(np.float32)
    return soup, np.arange(len(soup), dtype=np.int32).reshape(-1, 3)


@pytest.mark.parametrize("seed,jitter,min_dist", [(1, 0.0, 1e-4), (2, 3e-5, 1e-4), (3, 2e-4, 2e-3), (4, 0.0, 0.0)])
def test_flatten_vertices_matches_the_reference_text(seed, jitter, min_dist):
    rng = np.random.default_rng(seed)
    v, t = _mc_like_mesh(rng, 900, jitter)

    def run(kind):
        va, ta = oracle_py.flatten_vertices(v, t, min_dist, kind=kind)
        return {"n_verts": len(va), "n_tris": len(ta), "verts": va.view(np.uint32), "tris": ta}
    out = pinned(f"flatten_{seed}", run)
    assert min_dist == 0.0 or out["n_verts"] < len(v)


@pytest.mark.parametrize("seed,face_dist,min_neighbors", [(1, 0.02, 5), (2, 0.008, 3), (3, 0.05, 40)])
def test_cleanup_mesh_matches_the_reference_text(seed, face_dist, min_neighbors):
    rng = np.random.default_rng(seed)
    v, t = _mc_like_mesh(rng, 400, 0.0)
    v, t = oracle_py.flatten_vertices(v, t, 1e-4, kind="port")       # cleanupMesh runs on the welded mesh in the program (:707-712)

    def run(kind):
        va, ta = oracle_py.cleanup_mesh(v, t, face_dist, min_neighbors, kind=kind)
        return {"n_tris": len(ta), "verts": va.view(np.uint32), "tris": ta}
    assert pinned(f"cleanup_{seed}", run)["n_tris"] < len(t)
