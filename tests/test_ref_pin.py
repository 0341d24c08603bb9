"""Pins the CPU restatement (oracle/tsdf_oracle.cpp) against THE REFERENCE'S OWN SOURCES:
oracle/_ref/libcpu_tsdf_ref.so is the reference's src/lib/{octree,tsdf_volume_octree,
marching_cubes_tsdf_octree,tsdf_interface}.cpp + the reference headers compiled verbatim against
the Eigen/PCL compatibility layer in oracle/compat (oracle/Makefile `ref`).  Every decision the
reference's sources make — octree structure, split/prune history, per-node state, ray-march,
query arithmetic, mesher traversal, .vol layout — is compared bit for bit.

Each case computes its outputs through run(kind).  The restatement's outputs must reproduce the
digests of the reference build's outputs stored in tests/golden/ref_pins.json (written by
tools/make_ref_pins.py from oracle/_ref); where oracle/_ref is built, the reference's live outputs
must reproduce them as well."""
import json
import os

import numpy as np
import pytest

from cpu_tsdf_b200 import synth
from oracle import oracle_py
from oracle.oracle_py import OracleVolume
from tests.common import CFG_256, CFG_512, CFG_2048, digests, frames, nan_fixed, query_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PINS = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_pins.json")))["ref_pin"]
REF_LIB = oracle_py.REF_LIB


def pinned(key, run):
    """run("port") must reproduce the stored digests of run("reference"); returns the port's outputs"""
    got = run("port")
    assert digests(got) == PINS[key]
    if os.path.exists(REF_LIB):
        assert digests(run("reference")) == PINS[key]
    return got


def vol(kind, cfg, **kw):
    v = OracleVolume(kind=kind, **cfg, **kw)
    v.reset()
    return v


def nodes(d, rgb, var):
    out = {"keys": d["keys"], "split": d["split"], "dw": d["dw"].view(np.uint32)}
    if rgb:
        out["rgb"] = d["rgb"]
    if var:
        out["M"], out["ns"] = d["M"].view(np.uint32), d["ns"]
    return out


def run_defaults(kind):
    c = oracle_py.OrcConfig()
    oracle_py.load(kind).orc_default_config(c)
    out = {}
    for name, _ in oracle_py.OrcConfig._fields_:
        if name in ("num_threads",):
            continue
        va = getattr(c, name)
        out[name] = np.array(list(va)) if hasattr(va, "__len__") else va
    return out


INTEGRATE = [
    (CFG_256, synth.S1, 5, 9, True),
    (CFG_512, synth.S1, 4, 13, False),
    (CFG_2048, synth.S2, 2, 3, True),
]


def integrate_key(cfg, n, stride, color):
    return f"integrate_{cfg['xres']}_{n}_{stride}_{int(color)}"


def run_integrate(cfg, scene, n, stride, color):
    def run(kind):
        a = vol(kind, cfg, integrate_color=int(color))
        for pose, cloud in frames(scene, n, stride=stride, color=color, noise_seed=7, dropout=0.01):
            a.integrate(cloud, pose)
        return {"levels": np.array(a.levels()), **nodes(a.dump_nodes(), color, True)}
    return run


def run_cull_queries_render_mesh_vol(tmp_path):
    def run(kind):
        a = vol(kind, CFG_256, integrate_color=1)
        for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
            a.integrate(cloud, pose)
        out = {}
        for f in (0, 19, 44):
            m, k = a.frustum_cull(synth.orbit_pose(synth.S1, f, 100))
            out[f"cull{f}"], out[f"kept{f}"] = m, int(k)
        pts = query_points()
        for mode in (0, 1):
            q = a.query(pts, 7, mode)
            out[f"query{mode}_ok"] = q[3]
            for k in range(3):
                out[f"query{mode}_{k}"] = q[k][q[3]].view(np.uint32)
        pose = synth.orbit_pose(synth.S1, 10, 100)
        r, c = a.render(pose, 2, colored=True)
        out["render2_hits"] = int(np.isfinite(r[..., 2]).sum())
        out["render2_xyz"], out["render2_n"], out["render2_rgb"] = nan_fixed(r[..., :3]), nan_fixed(r[..., 4:7]), c
        out["render4"] = nan_fixed(a.render(pose, 4)[..., :7])
        for cm, wmin in ((0, 2.0), (1, 0.0), (2, 2.5)):
            v, col = a.mesh(wmin, cm)                    # same order too: both walk the octree depth-first
            out[f"mesh{cm}_n"], out[f"mesh{cm}"] = len(v), v
            out[f"mesh{cm}_rgb"] = col if col is not None else b"none"
        p = str(tmp_path / f"{kind}.vol")
        a.save(p)
        out["vol"] = open(p, "rb").read()
        return out
    return run


def run_rgb_normalized(tmp_path):
    def run(kind):
        a = vol(kind, CFG_256, integrate_color=1, color_mode=1)
        for pose, cloud in frames(synth.S1, 5, stride=7, color=True, noise_seed=5):
            a.integrate(cloud, pose)
        d = a.dump_nodes()
        out = {**nodes(d, True, True), "rgbn": d["rgbn"].view(np.uint32)}
        pose = synth.orbit_pose(synth.S1, 10, 100)
        r, c = a.render(pose, 4, colored=True)
        out["render4_xyz"], out["render4_rgb"] = nan_fixed(r[..., :3]), c
        v, col = a.mesh(0.0, 1)
        out["mesh_n"], out["mesh"], out["mesh_rgb"] = len(v), v.view(np.uint32), col
        p = str(tmp_path / f"{kind}.vol")
        out["save_rc"] = int(a.save(p))
        out["vol"] = open(p, "rb").read()
        # and the plain "RGB" mode is untouched by the new field
        c = vol(kind, CFG_256, integrate_color=1, color_mode=0)
        pose, cloud = next(frames(synth.S1, 1, color=True))
        c.integrate(cloud, pose)
        out["rgb_mode_has_rgbn"] = int("rgbn" in c.dump_nodes())
        out["rgb_mode_rgb"] = c.dump_nodes()["rgb"]
        return out
    return run


def _interp_points():
    rng = np.random.default_rng(3)
    vs = 3.0 / 256
    near = rng.normal(size=(3000, 3)); near *= 0.35 / np.linalg.norm(near, axis=1, keepdims=True); near += rng.normal(scale=0.01, size=near.shape)
    border = rng.uniform(-1.5, 1.5, (600, 3)); border[:, 0] = np.where(rng.random(600) < 0.5, -1.5 + vs * rng.uniform(0, 2, 600), 1.5 - vs * rng.uniform(0, 2, 600))
    outside = rng.uniform(-2.0, 2.0, (400, 3))
    nan = np.array([[np.nan, 0, 0], [0, 0, np.nan]])
    return np.concatenate([near, border, outside, nan]).astype(np.float32)


def run_get_tsdf_value(kind):
    a = vol(kind, CFG_256)
    for pose, cloud in frames(synth.S1, 3, stride=9, noise_seed=5):
        a.integrate(cloud, pose)
    pts = _interp_points()
    out = {}
    for vin in (True, False):
        v, ok = a.interpolate(pts, vin)
        out[f"ok{int(vin)}"], out[f"val{int(vin)}"] = ok, v.view(np.uint32)
        out[f"n_ok{int(vin)}"], out[f"n_nan{int(vin)}"] = int(ok.sum()), int(np.isnan(v).sum())
    return out


# ---- the tests ----------------------------------------------------------------------------------------------------------
def test_defaults_match_reference_constructor():
    pinned("defaults", run_defaults)


@pytest.mark.parametrize("cfg,scene,n,stride,color", INTEGRATE)
def test_integrate_structure_and_state(cfg, scene, n, stride, color):
    pinned(integrate_key(cfg, n, stride, color), run_integrate(cfg, scene, n, stride, color))


def test_cull_queries_render_mesh_vol(tmp_path):
    out = pinned("cull_queries_render_mesh_vol", run_cull_queries_render_mesh_vol(tmp_path))
    assert out["render2_hits"] > 20000
    assert min(out["mesh0_n"], out["mesh1_n"], out["mesh2_n"]) > 3000


def test_rgb_normalized_voxels_match_the_reference(tmp_path):
    """setColorMode("RGBNormalized") (tsdf_volume_octree.h:290, octree.cpp:378-433): normalised colour + intensity averages
    per node, getRGB's float -> uint8 conversions, and the serializer that writes the first byte of each float."""
    out = pinned("rgb_normalized", run_rgb_normalized(tmp_path))
    dw, rgbn = out["dw"].view(np.float32), out["rgbn"].view(np.float32)
    seen = dw[:, 1] > 0
    assert seen.sum() > 50000 and np.nanmax(rgbn[seen][:, 3]) > 100              # intensities are accumulated
    # unit colour direction wherever the pixel colour was not black (black gives 0/0 = NaN, as in the reference)
    rgb_dir = rgbn[seen][:, :3]; ok = np.isfinite(rgb_dir).all(1)
    assert ok.sum() > 0.9 * seen.sum() and np.abs(np.linalg.norm(rgb_dir[ok], axis=1) - 1).max() < 0.2
    assert out["render4_rgb"].any() and out["mesh_n"] > 3000 and out["save_rc"] == 0
    assert b"RGBNormalized\n#OCTREEBINARY\n" in out["vol"]
    assert out["rgb_mode_has_rgbn"] == 0


def test_get_tsdf_value_matches_the_reference():
    """getTSDFValue / interpolateTrilinearly (cpp:454-541; protected in the reference, reached through a derived accessor in the
    verbatim build): values bit-equal, NaN pattern and the in/out `valid` flag equal — inside, on the border layer, outside."""
    out = pinned("get_tsdf_value", run_get_tsdf_value)
    assert out["n_ok0"] == 0 and out["n_ok1"] > 500 and out["n_nan0"] > 100
