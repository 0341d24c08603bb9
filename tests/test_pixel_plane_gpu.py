"""The per-frame pixel plane against the CPU oracle, bit for bit.

k_front copies every pixel's z and colour word out of the caller's organized cloud into a plane of the handle, and the fast
observation of k_celltop_down and k_bricks reads the plane instead of the cloud.  These cases cover point layouts that no
other test combines: colour stored before xyz, a 48-byte stride, colour off (a 4-byte plane), and a sharded handle, whose
plane must hold every pixel although it fuses only its own coarse cells.  Each layout is fused through integrateCloudDevice
(one frame per call) and through integrateBatchDevice (one captured graph per batch)."""
import ctypes as C

import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_512, assert_same_nodes, frames

pytestmark = pytest.mark.gpu

NFRAMES = 4


def _stream(color):
    return list(frames(synth.S1, NFRAMES, stride=9, color=color, noise_seed=31, dropout=0.02))


def _repack(cloud, stride, xyz_off, rgba_off):
    """The same points (x, y, z bits and, with colour, the bgra word) at the given byte offsets of `stride`-byte records;
    the other bytes are filled with a pattern the engine must never read as data."""
    H, W, _ = cloud.shape
    out = np.full((H, W, stride // 4), 0x7FBADBAD, np.uint32)
    src = cloud.view(np.uint32)
    out[..., xyz_off // 4: xyz_off // 4 + 3] = src[..., 0:3]
    if rgba_off >= 0:
        out[..., rgba_off // 4] = src[..., 4]
    return np.ascontiguousarray(out)


def _engine(color, shard_rank=0, shard_count=1):
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=18, shard_rank=shard_rank, shard_count=shard_count)
    v.setResolution(CFG_512["xres"], CFG_512["yres"], CFG_512["zres"])
    v.setGridSize(CFG_512["xsize"], CFG_512["ysize"], CFG_512["zsize"])
    v.setCameraIntrinsics(525.0, 525.0, CAM.cx, CAM.cy)
    v.setIntegrateColor(color)
    v.reset()
    return v


def _pose(p):
    return np.ascontiguousarray(np.asarray(p, np.float64).reshape(4, 4))


def _fuse(v, dev, poses, stride, xyz_off, rgba_off, route):
    """integrateCloudDevice / integrateBatchDevice through the C ABI, which also takes the xyz offset"""
    import torch
    H, W = CAM.height, CAM.width
    if route == "frames":
        for d, p in zip(dev, poses):
            pp = _pose(p)
            v._check(v._lib.b200tsdf_integrate_device(v._h, C.c_void_p(d.data_ptr()), stride, xyz_off, rgba_off, W, H, pp.ctypes.data))
    else:
        for lo, hi in ((0, 3), (3, len(dev))):        # a captured graph, then the other half of the record ring
            arr = (C.c_void_p * (hi - lo))(*[C.c_void_p(d.data_ptr()) for d in dev[lo:hi]])
            ps = np.ascontiguousarray(np.stack([_pose(p) for p in poses[lo:hi]]))
            v._check(v._lib.b200tsdf_integrate_batch_device(v._h, hi - lo, arr, stride, xyz_off, rgba_off, W, H, ps.ctypes.data))
    v.sync()
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def oracle_color():
    fs = _stream(True)
    o = OracleVolume(**CFG_512, integrate_color=1)
    o.reset()
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    return fs, o.dump_nodes(), o.stats().n_add_observation


@pytest.fixture(scope="module")
def oracle_depth():
    fs = _stream(False)
    o = OracleVolume(**CFG_512)
    o.reset()
    for pose, cloud in fs:
        o.integrate(cloud, pose)
    return fs, o.dump_nodes(), o.stats().n_add_observation


LAYOUTS = {
    # name: (colour, stride, xyz_off, rgba_off)
    "rgba_before_xyz": (True, 32, 16, 0),
    "stride48": (True, 48, 8, 40),
    "colour_off": (False, 20, 8, -1),
}


@pytest.mark.parametrize("route", ["frames", "batch"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layout_matches_the_oracle(layout, route, oracle_color, oracle_depth):
    import torch
    color, stride, xyz_off, rgba_off = LAYOUTS[layout]
    fs, ref, n_upd = oracle_color if color else oracle_depth
    dev = [torch.from_numpy(_repack(c, stride, xyz_off, rgba_off)).cuda() for _, c in fs]
    v = _engine(color)
    _fuse(v, dev, [p for p, _ in fs], stride, xyz_off, rgba_off, route)
    assert_same_nodes(ref, v.download_nodes(), rgb=color)
    assert v.stats().n_updates == n_upd


@pytest.mark.parametrize("route", ["frames", "batch"])
def test_sharded_handles_see_every_pixel(route, oracle_color):
    """Two shards of one volume on one device: a shard fuses only its own coarse cells, but the observations of its nodes read
    pixels whose points fall in the other shard's cells.  Each shard's nodes equal the oracle's nodes of the cells it owns."""
    import torch
    from tests.shard_worker import cell_owner
    fs, ref, n_upd = oracle_color
    stride, xyz_off, rgba_off = 48, 8, 40
    dev = [torch.from_numpy(_repack(c, stride, xyz_off, rgba_off)).cuda() for _, c in fs]

    def owners(keys, C0):
        cells, inv = np.unique(keys[:, 1:] >> (keys[:, 0:1] - C0), axis=0, return_inverse=True)
        return np.array([cell_owner(*c, 2) for c in cells])[inv.reshape(-1)]

    C0 = None
    for r in range(2):
        v = _engine(True, shard_rank=r, shard_count=2)
        _fuse(v, dev, [p for p, _ in fs], stride, xyz_off, rgba_off, route)
        if C0 is None:
            C0 = v.stats().coarse_level
            owner = owners(ref["keys"], C0)
        d = v.download_nodes()
        own = owners(d["keys"], C0) == r
        assert own.any()
        assert np.array_equal(d["keys"][own], ref["keys"][owner == r])
        assert np.array_equal(d["dw"][own].view(np.uint32), ref["dw"][owner == r].view(np.uint32))
        assert np.array_equal(d["rgb"][own], ref["rgb"][owner == r])
        assert np.array_equal(d["split"][own], ref["split"][owner == r])
        del v
