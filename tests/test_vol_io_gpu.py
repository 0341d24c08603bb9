""".vol save and load through the device (DESIGN.md §3e) on a real H100.

* Save parity: the device writer's bytes equal the reference's save and the host writer's (debug_flags bit 2) on the same
  handle, over grid shapes, colour modes, track_variance, writes through setContainingVoxelsData, a fresh volume and a shard.
* Pin cases: the dynamic scenes K1-K6 (pruning and re-splitting) and the exact-tie cases E1-E5 save the reference's bytes
  on both writers, and the device parser (b200tsdf_load_path) takes those files back.
* Round trips: the parallel parser and the host loader rebuild the same volume from the files of the restatement and of
  the reference's own build (oracle/_ref); 20 further frames fused into both stay equal to each other and to the reference,
  and so do render, mesh and leaf lists.
* Fallback: malformed or unusual bodies give the host loader's result on both paths, through files and device images.
* Route check: a loaded {d, w} outside the fast route's domain moves the next integrate to the general kernel.
* Device images: saveDevice / loadDevice against save / load, the size query and the capacity check."""
import os
import struct

import numpy as np
import pytest
import torch

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle import leaves_py, oracle_py
from oracle.edits_py import EditsOracleVolume
from oracle.oracle_py import OracleVolume
from tests import dynamic_cases, general_cases
from tests.common import CAM, CFG_256, CFG_512, CFG_2048, assert_same_nodes, frames

pytestmark = pytest.mark.gpu

HOST_IO = 4          # debug_flags bit 2: the host writer and the host loader


def cfg_of(res, size, cell=None):
    c = dict(xres=res, yres=res, zres=res, xsize=size, ysize=size, zsize=size, cx=CAM.cx, cy=CAM.cy)
    if cell:
        c.update(max_cell_x=cell, max_cell_y=cell, max_cell_z=cell)
    return c


def engine(cfg, pool_log2=17, color=False, var=False, mode=None, flags=0, **kw):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, track_variance=var, **kw)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg["xsize"], cfg["ysize"], cfg["zsize"])
    v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy)
    if "max_cell_x" in cfg:
        v.setMaxVoxelSize(cfg["max_cell_x"], cfg["max_cell_y"], cfg["max_cell_z"])
    if color:
        v.setIntegrateColor(True)
    if mode:
        v.setColorMode(mode)
    set_flags(v, flags)
    v.reset()
    return v


def set_flags(v, flags):
    v._cfg.debug_flags = flags
    v._push()


def both_saves(v, tmp_path, tag):
    """the device writer's bytes and the host writer's, from one handle"""
    pd, ph = tmp_path / f"{tag}_dev.vol", tmp_path / f"{tag}_host.vol"
    keep = v._cfg.debug_flags
    set_flags(v, keep & ~HOST_IO); v.save(str(pd))
    set_flags(v, keep | HOST_IO); v.save(str(ph))
    set_flags(v, keep)
    return pd.read_bytes(), ph.read_bytes()


def nodes(v):
    return v.download_nodes()


def same_volume(a, b, var=False):
    na, nb = nodes(a), nodes(b)
    assert_same_nodes(na, nb, rgb=True, var=var)
    assert np.array_equal(na["split"], nb["split"])
    assert a.isEmpty() == b.isEmpty()


def loaded(path, flags, var=False, pool_log2=17, path_is=None):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2, track_variance=var)
    set_flags(v, flags)
    v.load(str(path))
    if path_is:
        assert v.loadPath() == path_is
    return v


# ---- save parity -----------------------------------------------------------------------------------------------------------
# track_variance on every shape: the reference's files carry M_ / nsample_, which the engine keeps only with it
SHAPES = [
    ("256_rgb", CFG_256, dict(color=True), synth.S1),
    ("512", CFG_512, {}, synth.S1),
    ("2048_rgb", CFG_2048, dict(color=True), synth.S2),
    ("128_c0.5", cfg_of(128, 3.0, 0.5), {}, None),
    ("1024_c0.5", cfg_of(1024, 3.0, 0.5), {}, None),
    ("256_2.7_c0.3", cfg_of(256, 2.7, 0.3), {}, None),
    ("512_12_c0.5", cfg_of(512, 12.0, 0.5), {}, None),
]


@pytest.mark.parametrize("name,cfg,kw,scene", SHAPES, ids=[s[0] for s in SHAPES])
def test_save_parity(tmp_path, name, cfg, kw, scene):
    scene = scene or synth.Scene(room_half=min(1.3, cfg["xsize"] * 0.45), cam_radius=0.8)
    o = OracleVolume(**cfg, **({"integrate_color": 1} if kw.get("color") else {}))
    o.reset()
    e = engine(cfg, 18, var=True, **kw)
    for pose, cloud in frames(scene, 3, stride=7, color=kw.get("color", False), noise_seed=5):
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    dev, host = both_saves(e, tmp_path, name)
    po = tmp_path / "o.vol"
    assert o.save(str(po)) == 0
    assert dev == po.read_bytes()
    assert dev == host


def test_save_parity_fresh_rgbn_edits_and_shards(tmp_path):
    fresh = engine(CFG_256, 14, color=True)
    dev, host = both_saves(fresh, tmp_path, "fresh")
    o = OracleVolume(**CFG_256, integrate_color=1); o.reset()
    po = tmp_path / "o.vol"; o.save(str(po))
    assert dev == host == po.read_bytes()

    rgbn = engine(CFG_256, 17, color=True, mode="RGBNormalized")
    for pose, cloud in frames(synth.S1, 2, stride=9, color=True, noise_seed=3):
        rgbn.integrateCloud(cloud, None, pose)
    dev, host = both_saves(rgbn, tmp_path, "rgbn")
    assert dev == host and len(dev) > 100000

    ed = engine(CFG_512, 18, color=True, var=True)
    oe = EditsOracleVolume(**CFG_512, integrate_color=1); oe.reset()
    for pose, cloud in frames(synth.S1, 2, stride=9, color=True, noise_seed=4):
        ed.integrateCloud(cloud, None, pose); oe.integrate(cloud, pose)
    rng = np.random.default_rng(7)
    pts = rng.uniform(-1.2, 1.2, (4000, 3)).astype(np.float32)
    d, w = np.full(4000, 0.25, np.float32), np.full(4000, 3.0, np.float32)
    st = ed.setContainingVoxelsData(pts, d, w)
    assert (st == 0).sum() > 1000 and np.array_equal(st, oe.set_containing_voxels(pts, d, w))
    dev, host = both_saves(ed, tmp_path, "edits")
    assert oe.save(str(po)) == 0
    assert dev == host == po.read_bytes()

    for r in range(2):
        sh = engine(CFG_256, 16, shard_rank=r, shard_count=2)
        for pose, cloud in frames(synth.S1, 2, stride=11, noise_seed=21):
            sh.integrateCloud(cloud, None, pose)
        dev, host = both_saves(sh, tmp_path, f"shard{r}")
        assert dev == host


# ---- the pin cases: pruning, re-splitting, exact ties -----------------------------------------------------------------------
PIN_CASES = [dynamic_cases.CASES[k] for k in ("K1", "K2", "K3", "K4", "K5", "K6")] + \
            [general_cases.CASES[k] for k in ("E1", "E2", "E3", "E4", "E5")]


@pytest.mark.parametrize("case", PIN_CASES, ids=[c.id for c in PIN_CASES])
def test_pin_cases_save_and_load(tmp_path, case):
    pool = {256: 17, 512: 18, 2048: 18, 4096: 19}[case.res]
    e = pkg.TSDFVolumeOctree(device=0, pool_log2=pool, track_variance=True)
    for k, x in case.config().items():
        setattr(e._cfg, k, x)
    e._push(); e.reset()
    o = OracleVolume(**case.config()); o.reset()
    for pose, cloud in case.frames():
        o.integrate(cloud, pose); e.integrateCloud(cloud, None, pose)
    dev, host = both_saves(e, tmp_path, case.id)
    po = tmp_path / "o.vol"
    assert o.save(str(po)) == 0
    assert dev == host == po.read_bytes()
    if getattr(case, "color_mode", 0) == 0:             # (RGBNormalized files are refused by load(), as the reference's are)
        a = loaded(tmp_path / f"{case.id}_dev.vol", 0, True, pool, path_is="device")
        b = loaded(tmp_path / f"{case.id}_dev.vol", HOST_IO, True, pool, path_is="host")
        same_volume(a, b, var=True)
        assert_same_nodes(o.dump_nodes(), nodes(a), rgb=case.color, var=True)


# ---- round trips ---------------------------------------------------------------------------------------------------------
HAVE_REF = os.path.exists(oracle_py.REF_LIB) and os.path.exists(leaves_py.REF_LIB)
TRIPS = [("256_rgb_var", CFG_256, True, True, synth.S1, "port"), ("512", CFG_512, False, False, synth.S1, "port"),
         ("2048_rgb", CFG_2048, True, False, synth.S2, "port"), ("256_rgb_var_ref", CFG_256, True, True, synth.S1, "reference"),
         ("512_ref", CFG_512, False, False, synth.S1, "reference")]


def leaf_lists(v):
    return v.getVoxelCenters(-1).view(np.uint32), v.getOccupiedVoxelIndices()


@pytest.mark.parametrize("name,cfg,color,var,scene,kind", TRIPS, ids=[t[0] for t in TRIPS])
def test_round_trip_reference_files(tmp_path, name, cfg, color, var, scene, kind):
    if kind == "reference" and not HAVE_REF:
        pytest.skip("the reference's own build (oracle/_ref) is not built")
    o = leaves_py.LeavesOracleVolume(kind=kind, **cfg, **({"integrate_color": 1} if color else {}))
    o.reset()
    fr = list(frames(scene, 23, stride=4, color=color, noise_seed=9))
    for pose, cloud in fr[:3]:
        o.integrate(cloud, pose)
    pa = tmp_path / "a.vol"
    assert o.save(str(pa)) == 0
    dev, host = loaded(pa, 0, var, 18, path_is="device"), loaded(pa, HOST_IO, var, 18, path_is="host")
    same_volume(dev, host, var)
    assert_same_nodes(o.dump_nodes(), nodes(dev), rgb=color, var=var)
    gen = loaded(pa, 1, var, 18, path_is="device")    # the general kernel as well
    for pose, cloud in fr[3:]:
        o.integrate(cloud, pose)
        for v in (dev, host, gen):
            v.integrateCloud(cloud, None, pose)
    ref = o.dump_nodes()
    for v in (dev, host, gen):
        assert_same_nodes(ref, nodes(v), rgb=color, var=var)
    pose = fr[10][0]
    ra, rb = o.render(pose, 2), dev.renderView(pose, 2)
    assert np.array_equal(ra[..., :3], rb[..., :3], equal_nan=True) and np.array_equal(ra[..., 4:7], rb[..., 4:7], equal_nan=True)
    mc = pkg.MarchingCubesTSDFOctree(); mc.setInputTSDF(dev); mc.setMinWeight(0.0)
    vb, _, _ = mc.reconstruct()
    va, _ = o.mesh(0.0, 0)
    assert np.array_equal(np.asarray(va).view(np.uint32), np.asarray(vb).reshape(-1, 3).view(np.uint32))
    centres, occupied = leaf_lists(dev)
    assert np.array_equal(centres, o.voxel_centers(-1).view(np.uint32)) and np.array_equal(occupied, o.occupied_voxel_indices())
    b, c = tmp_path / "b.vol", tmp_path / "c.vol"
    dev.save(str(b)); host.save(str(c))
    assert b.read_bytes() == c.read_bytes()
    if var:                                            # M_ / nsample_ are in the engine's files only with track_variance
        assert o.save(str(pa)) == 0 and b.read_bytes() == pa.read_bytes()


# ---- fallback ------------------------------------------------------------------------------------------------------------
def body_offset(raw):
    return raw.index(b"#OCTREEBINARY\n") + len(b"#OCTREEBINARY\n") + 36


def outcome(fn):
    try:
        v = fn()
    except pkg.B200Error as ex:
        return ("error", str(ex).split(": ")[-1])
    return ("ok", v)


def test_malformed_and_unusual_bodies(tmp_path):
    e = engine(CFG_256, 17)
    for pose, cloud in frames(synth.S1, 2, stride=9, noise_seed=6):
        e.integrateCloud(cloud, None, pose)
    src = tmp_path / "src.vol"; e.save(str(src))
    raw = src.read_bytes()
    off, R = body_offset(raw), 40
    n = (len(raw) - off) // R

    def rec_field(buf, i, at, fmt, val):
        b = bytearray(buf)
        struct.pack_into(fmt, b, off + i * R + at, val)
        return bytes(b)

    sizes = [struct.unpack_from("<f", raw, off + i * R + 20)[0] for i in range(n)]
    finest = min(range(n), key=lambda i: sizes[i])
    cx0 = struct.unpack_from("<f", raw, off + finest * R + 8)[0]
    cases = {
        "truncated": raw[:-20],
        "nchild3": rec_field(raw, 5, 32, "<Q", 3),
        "shallow": rec_field(raw, 0, 32, "<Q", 0),
        "deep": rec_field(raw, finest, 32, "<Q", 8),
        "ulp": rec_field(raw, finest, 8, "<f", float(np.nextafter(np.float32(cx0), np.float32(np.inf)))),
        "trailing": raw + b"\x01" * 57,
    }
    for name, buf in cases.items():
        p = tmp_path / f"{name}.vol"; p.write_bytes(buf)
        a = outcome(lambda: loaded(p, 0, path_is="device" if name == "trailing" else "host"))
        b = outcome(lambda: loaded(p, HOST_IO, path_is="host"))

        def from_device():
            v = pkg.TSDFVolumeOctree(device=0, pool_log2=17)
            t = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
            torch.cuda.synchronize()
            v.loadDevice(t.data_ptr(), t.numel())
            assert v.loadPath() == ("device" if name == "trailing" else "host")
            return v
        c = outcome(from_device)
        assert a[0] == b[0] == c[0], (name, a, b, c)
        if a[0] == "error":
            assert a[1] == b[1] == c[1], name
        else:
            same_volume(a[1], b[1]); same_volume(a[1], c[1])
    assert outcome(lambda: loaded(tmp_path / "truncated.vol", 0))[0] == "error"
    assert outcome(lambda: loaded(tmp_path / "trailing.vol", 0))[0] == "ok"
    same_volume(loaded(tmp_path / "trailing.vol", 0), loaded(src, 0))


# ---- route check ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,w", [(0.25, -0.5), (2.0 ** 40, 1.0)], ids=["w=-0.5", "d=2^40"])
def test_out_of_domain_values_take_the_general_kernel(tmp_path, d, w):
    e = engine(CFG_256, 17, var=True)
    o = EditsOracleVolume(**CFG_256); o.reset()
    fr = list(frames(synth.S1, 5, stride=7, noise_seed=8))
    for pose, cloud in fr[:2]:
        e.integrateCloud(cloud, None, pose); o.integrate(cloud, pose)
    src = tmp_path / "src.vol"; e.save(str(src))
    raw = src.read_bytes()
    off, R = body_offset(raw), 40
    leaf = np.array([struct.unpack_from("<3f", raw, len(raw) - R + 8)], np.float32)     # the last record: a stored leaf
    for v in (e, o):                                   # the file and the reference both hold the value at that leaf
        st = v.setContainingVoxelsData(leaf, np.float32(d), np.float32(w)) if v is e else v.set_containing_voxels(leaf, d, w)
        assert st.tolist() == [0]
    p = tmp_path / "ood.vol"; e.save(str(p))
    assert o.save(str(src)) == 0 and src.read_bytes() == p.read_bytes()
    clean = engine(CFG_256, 17)
    for pose, cloud in fr[:3]:
        clean.integrateCloud(cloud, None, pose)
    clean.save(str(src))
    clean = loaded(src, 0, path_is="device")
    clean.integrateCloud(fr[3][1], None, fr[3][0])
    assert clean.stats().n_block_visits > 0              # a file fusion wrote keeps the fast route
    vols = [loaded(p, 0, True, path_is="device"), loaded(p, HOST_IO, True, path_is="host"), loaded(p, 1, True)]
    for pose, cloud in fr[2:]:
        o.integrate(cloud, pose)
        for v in vols:
            v.integrateCloud(cloud, None, pose)
            assert v.stats().n_block_visits == 0
    for v in vols:
        assert_same_nodes(o.dump_nodes(), nodes(v), var=True)


# ---- device images -------------------------------------------------------------------------------------------------------
def test_device_images(tmp_path):
    e = engine(CFG_512, 18, color=True)
    for pose, cloud in frames(synth.S1, 3, stride=9, color=True, noise_seed=2):
        e.integrateCloud(cloud, None, pose)
    p = tmp_path / "a.vol"; e.save(str(p))
    raw = p.read_bytes()
    n = e.saveDevice()
    assert n == len(raw)
    buf = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with pytest.raises(pkg.B200Error, match="too small"):
        e.saveDevice(buf.data_ptr(), n - 1)
    assert bool((buf == 0xAB).all())                  # nothing written
    assert e.saveDevice(buf.data_ptr(), n + 64) == n
    img = buf[:n].cpu().numpy().tobytes()
    assert img == raw and bool((buf[n:] == 0xAB).all())
    for flags in (0, HOST_IO):
        v = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
        set_flags(v, flags)
        v.loadDevice(buf.data_ptr(), n)
        assert v.loadPath() == ("device" if flags == 0 else "host")
        same_volume(v, e)
        assert v.getResolution() == (512, 512, 512)
    # a pool too small for the file fails as the host loader fails
    small = [outcome(lambda f=f: loaded(p, f, pool_log2=8)) for f in (0, HOST_IO)]
    assert small[0][0] == small[1][0] == "error" and small[0][1] == small[1][1] and "pool" in small[0][1]


def test_stream_2048_save_and_load(tmp_path):
    e = engine(CFG_2048, 20, color=True)
    for f in range(30):
        pose = synth.orbit_pose(synth.S2, f, 100)
        e.integrateCloud(synth.make_frame(synth.S2, pose, CAM, color=True, noise_seed=77, frame=f), None, pose)
    dev, host = both_saves(e, tmp_path, "s2048")
    assert dev == host and len(dev) > 50_000_000
    a = loaded(tmp_path / "s2048_dev.vol", 0, pool_log2=20, path_is="device")
    b = loaded(tmp_path / "s2048_dev.vol", HOST_IO, pool_log2=20, path_is="host")
    same_volume(a, b)
    same_volume(a, e)
