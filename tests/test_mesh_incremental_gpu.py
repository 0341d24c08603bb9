"""Incremental meshing on the engine (DESIGN.md §3g): IncrementalMesh.update() against reconstructDevice, bit for bit, after
every frame, batch or write, on every integrate route and across whole-volume changes; the device's change mask against the
host emulation's; the calls that must not move the epoch; and the argument checks of reconstructCellsDevice."""
import numpy as np
import pytest
import torch

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from tests import dynamic_cases
from tests.common import CFG_256, frames
from tests.emu import cells_py
from tests.emu.cells_py import CellsEmuVolume

pytestmark = pytest.mark.gpu

GT = np.array([[0.0, -0.8, 0.6, 0.25], [1.0, 0.0, 0.0, -1.5], [0.0, 0.6, 0.8, 3.0], [0, 0, 0, 1]])


def _engine(cfg, pool_log2=18, **extra):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=pool_log2)
    for k, x in {**cfg, **extra}.items():
        setattr(v._cfg, k, x)
    v._push()
    v.reset()
    return v


def full_mesh(vol, w_min, color_mode):
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(vol); mc.setMinWeight(w_min)
    mc.setColorByRGB(color_mode == 1); mc.setColorByConfidence(color_mode == 2)
    n = mc.reconstructDevice()
    v = torch.empty((max(n, 1), 3), dtype=torch.float32, device="cuda:0")
    c = torch.empty((max(n, 1), 3), dtype=torch.uint8, device="cuda:0")
    assert mc.reconstructDevice(v.data_ptr(), n, c.data_ptr() if color_mode else None) == n
    return v[:n], (c[:n] if color_mode else None)


def same(inc, vol):
    got_v, got_c = inc.update()
    want_v, want_c = full_mesh(vol, inc.w_min, inc.color_mode)
    assert got_v.shape == want_v.shape, (got_v.shape, want_v.shape)
    assert torch.equal(got_v.view(torch.int32), want_v.view(torch.int32)), "vertices differ from reconstructDevice"
    if inc.color_mode:
        assert torch.equal(got_c, want_c), "colours differ from reconstructDevice"
    else:
        assert got_c is None
    return inc.cells_remeshed


def test_rgb_stream_256_every_frame():
    vol = _engine(CFG_256, integrate_color=1)
    incs = [pkg.IncrementalMesh(vol, 2.0, 1), pkg.IncrementalMesh(vol, 0.0, 2)]
    for inc in incs:
        same(inc, vol)
    partial = 0
    for pose, cloud in frames(synth.S1, 8, stride=7, color=True, noise_seed=5):
        vol.integrateCloud(cloud, None, pose)
        for inc in incs:
            partial += same(inc, vol) < vol.changedCells(0)[1].size
    assert partial > 0, "no update re-meshed only part of the cells"


@pytest.mark.parametrize("cid", ["K1", "K2", "K3", "K4", "K5", "K6"])
def test_dynamic_cases(cid):
    case = dynamic_cases.CASES[cid]
    vol = _engine(case.config(), pool_log2=18 if case.res < 2048 else 20)
    inc = pkg.IncrementalMesh(vol, 0.0, 1 if case.color else 2)
    same(inc, vol)
    for pose, cloud in case.frames():
        vol.integrateCloud(cloud, None, pose)
        same(inc, vol)


def _device_clouds(clouds):
    return [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in clouds]


def test_routes_and_switches_without_sync():
    """integrateCloud, integrateCloudDevice, integrateCloudAsync, integrateBatchDevice and integrateUnorganizedBatchDevice in
    turn, with no sync between a route switch and the update"""
    vol = _engine(CFG_256, integrate_color=1)
    inc = pkg.IncrementalMesh(vol, 2.0, 1)
    same(inc, vol)
    fr = list(frames(synth.S1, 12, stride=5, color=True, noise_seed=9))
    poses = [p for p, _ in fr]
    clouds = [c for _, c in fr]
    d = _device_clouds(clouds)
    H, W, nf = clouds[0].shape
    vol.integrateCloud(clouds[0], None, poses[0]); same(inc, vol)
    vol.integrateCloudDevice(d[1].data_ptr(), H, W, nf * 4, poses[1], 16); same(inc, vol)
    pinned = torch.from_numpy(np.ascontiguousarray(clouds[2])).pin_memory()
    vol.integrateCloudAsync(pinned.data_ptr(), H, W, nf * 4, poses[2], 16); same(inc, vol)
    vol.integrateBatchDevice([t.data_ptr() for t in d[3:6]], H, W, nf * 4, poses[3:6], 16); same(inc, vol)
    vol.integrateCloudDevice(d[6].data_ptr(), H, W, nf * 4, poses[6], 16)
    vol.integrateBatchDevice([t.data_ptr() for t in d[7:9]], H, W, nf * 4, poses[7:9], 16); same(inc, vol)
    # unorganised clouds: the organised frames' valid points
    pts = []
    for c in clouds[9:12]:
        q = c.reshape(-1, nf)
        pts.append(torch.from_numpy(np.ascontiguousarray(q[~np.isnan(q[:, 2])])).cuda())
    vol.integrateUnorganizedBatchDevice([t.data_ptr() for t in pts], [len(t) for t in pts], nf * 4, poses[9:12], 16)
    same(inc, vol)


def test_writes_load_reset_transform_and_mode_changes(tmp_path):
    vol = _engine(CFG_256, integrate_color=1)
    inc = pkg.IncrementalMesh(vol, 2.0, 1)
    fr = list(frames(synth.S1, 8, stride=9, color=True, noise_seed=4))
    for pose, cloud in fr[:3]:
        vol.integrateCloud(cloud, None, pose)
    same(inc, vol)
    rng = np.random.default_rng(3)
    pts = rng.uniform(-0.5, 0.5, (2000, 3)).astype(np.float32)
    vol.setContainingVoxelsData(pts, rng.uniform(-0.9, 0.9, 2000).astype(np.float32), np.full(2000, 5.0, np.float32))
    same(inc, vol)
    vol.integrateCloud(fr[3][1], None, fr[3][0]); same(inc, vol)
    vol.save(str(tmp_path / "a.vol"))
    vol.integrateCloud(fr[4][1], None, fr[4][0]); same(inc, vol)
    vol.load(str(tmp_path / "a.vol")); same(inc, vol)
    nbytes = vol.saveDevice()
    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    vol.saveDevice(buf.data_ptr(), nbytes)
    vol.integrateCloud(fr[5][1], None, fr[5][0]); same(inc, vol)
    vol.loadDevice(buf.data_ptr(), nbytes); same(inc, vol)
    vol.setGlobalTransform(GT); same(inc, vol)
    vol.integrateCloud(fr[6][1], None, fr[6][0]); same(inc, vol)
    inc.w_min = 0.0; same(inc, vol)
    inc.color_mode = 2; same(inc, vol)
    inc.color_mode = 0; same(inc, vol)
    vol.reset(); same(inc, vol)
    vol.integrateCloud(fr[7][1], None, fr[7][0]); same(inc, vol)


@pytest.mark.parametrize("cid", ["K1", "K6"])
def test_mask_equals_emulation(cid):
    case = dynamic_cases.CASES[cid]
    vol = _engine(case.config())
    emu = CellsEmuVolume(**case.config(), pool_log2=17)
    emu.reset()
    since_d, since_e = vol.changedCells(0)[0], cells_py.changed_cells(emu, 0)[0]
    for pose, cloud in case.frames():
        vol.integrateCloud(cloud, None, pose)
        emu.integrate(cloud, pose)
        now_d, mask_d = vol.changedCells(since_d)
        now_e, mask_e = cells_py.changed_cells(emu, since_e)
        assert now_d - since_d == now_e - since_e == 1
        assert np.array_equal(mask_d, mask_e)
        since_d, since_e = now_d, now_e


def test_no_change_calls(tmp_path):
    vol = _engine(CFG_256, integrate_color=1, pool_log2=16)
    for pose, cloud in frames(synth.S1, 3, stride=9, color=True, noise_seed=4):
        vol.integrateCloud(cloud, None, pose)
    now, _ = vol.changedCells(0)
    vol.resizePool(18)
    vol.save(str(tmp_path / "b.vol"))
    vol.saveDevice()
    vol.renderView(synth.orbit_pose(synth.S1, 0, 100), 4)
    vol.getFxn(np.zeros((4, 3), np.float32))
    pkg.MarchingCubesTSDFOctree().setInputTSDF(vol)
    with pytest.raises(pkg.B200Error):
        vol.resizePool(3)                                                  # refused: outside [8, 26]
    with pytest.raises(pkg.B200Error):
        vol.integrateCloud(np.zeros((2, 2, 8), np.float32), None, np.eye(4))   # refused: wrong image size
    vol.setContainingVoxelsData(np.full((3, 3), 9.0, np.float32), np.zeros(3, np.float32), np.ones(3, np.float32))  # outside: no node
    now2, mask = vol.changedCells(now)
    assert now2 == now and not mask.any()
    vol._push()                                                            # the same configuration again: no change
    now3, mask = vol.changedCells(now)
    assert now3 == now and not mask.any()


def test_reconstruct_cells_device_arguments():
    vol = pkg.TSDFVolumeOctree(device=0, pool_log2=16)
    mc = pkg.MarchingCubesTSDFOctree(); mc.setInputTSDF(vol); mc.setColorByRGB(True)
    for k, x in CFG_256.items():
        setattr(vol._cfg, k, x)
    vol._cfg.integrate_color = 1
    vol._push()
    with pytest.raises(pkg.B200Error, match=r"code -4|before reset"):
        vol.changedCells(0)
    vol.reset()
    for pose, cloud in frames(synth.S1, 3, stride=9, color=True, noise_seed=4):
        vol.integrateCloud(cloud, None, pose)
    ncells = vol.changedCells(0)[1].size
    n_all, counts = mc.reconstructCellsDevice(None)
    assert n_all == mc.reconstructDevice() and counts.sum() == n_all and counts.size == ncells
    mask = np.zeros(ncells, np.uint8); mask[np.flatnonzero(counts)[::2]] = 1
    n, cnt = mc.reconstructCellsDevice(mask)
    assert n == counts[mask != 0].sum() and np.array_equal(cnt, np.where(mask != 0, counts, 0))
    buf = torch.empty((n_all + 1, 3), dtype=torch.float32, device="cuda:0")
    rgb = torch.empty((n_all + 1, 3), dtype=torch.uint8, device="cuda:0")
    with pytest.raises(pkg.B200Error):
        mc.reconstructCellsDevice(mask, buf.data_ptr(), n - 1, rgb.data_ptr())
    with pytest.raises(pkg.B200Error):
        mc.reconstructCellsDevice(mask, buf.data_ptr() + 2, n, rgb.data_ptr())
    assert mc.reconstructCellsDevice(None, buf.data_ptr(), n_all, rgb.data_ptr())[0] == n_all
    want_v, want_c = full_mesh(vol, mc.w_min_, 1)
    assert torch.equal(buf[:n_all].view(torch.int32), want_v.view(torch.int32)) and torch.equal(rgb[:n_all], want_c)
    # a shard refuses both calls
    sh = pkg.TSDFVolumeOctree(device=0, pool_log2=16)
    for k, x in CFG_256.items():
        setattr(sh._cfg, k, x)
    sh._cfg.shard_count = 2; sh._cfg.shard_rank = 0
    sh._push(); sh.reset()
    with pytest.raises(pkg.B200Error, match="shard"):
        sh.changedCells(0)
    ms = pkg.MarchingCubesTSDFOctree(); ms.setInputTSDF(sh)
    with pytest.raises(pkg.B200Error, match="shard"):
        ms.reconstructCellsDevice(None)


def test_cpp_shim_cells(engine_lib, tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    libdir = os.path.dirname(engine_lib)
    exe = os.path.join(str(tmp_path), "shim_cells")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-O1", os.path.join(root, "tests", "cpp", "shim_cells.cpp"), "-o", exe, "-I/usr/local/cuda/include",
                    f"-L{libdir}", "-lb200tsdf", f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-lcudart",
                    "-Wl,-rpath,/usr/local/cuda/lib64"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "mesh:" in r.stdout
