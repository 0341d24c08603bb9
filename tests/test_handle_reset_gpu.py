"""reset() either installs the new volume whole or leaves the handle without one.

A reset whose device memory cannot be had (here the node array of a 2^26-brick pool, about 313 GB, which fails at once)
returns B200TSDF_ENOMEM, and every call that needs a volume then returns B200TSDF_ESTATE until a reset succeeds; that reset
builds the same volume as a handle that never failed.  A configuration reset() refuses (B200TSDF_EINVAL) leaves the previous
volume as it was."""
import numpy as np
import pytest

import cpu_tsdf_b200 as pkg
from cpu_tsdf_b200 import synth
from tests.common import CAM, CFG_512, frames

pytestmark = pytest.mark.gpu

ENOMEM, ESTATE, EINVAL = -4, -5, -1
FRAMES = list(frames(synth.S1, 2, stride=5, noise_seed=3))
PTS = np.random.default_rng(7).uniform(-0.6, 0.6, (512, 3)).astype(np.float32)


def _volume():
    v = pkg.TSDFVolumeOctree(device=0, pool_log2=18)
    v.setResolution(CFG_512["xres"], CFG_512["yres"], CFG_512["zres"])
    v.setGridSize(CFG_512["xsize"], CFG_512["ysize"], CFG_512["zsize"])
    v.setCameraIntrinsics(CAM.fx, CAM.fy, CAM.cx, CAM.cy)
    v.reset()
    return v


def _fuse(v):
    for pose, cloud in FRAMES:
        v.integrateCloud(cloud, None, pose)
    v.sync()


def _assert_same_nodes(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


def _raises(code, call):
    with pytest.raises(pkg.B200Error, match=rf"\(code {code}\)"):
        call()


def test_failed_reset_leaves_no_volume_until_a_reset_succeeds(tmp_path):
    import torch
    fresh = _volume()
    _fuse(fresh)
    v = _volume()
    _fuse(v)
    v._cfg.pool_log2 = 26
    v._push()
    _raises(ENOMEM, v.reset)

    pose, cloud = FRAMES[0]
    H, W, nf = cloud.shape
    d_cloud = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    mc = pkg.MarchingCubesTSDFOctree()
    mc.setInputTSDF(v)
    calls = {
        "integrateCloud": lambda: v.integrateCloud(cloud, None, pose),
        "integrateBatchDevice": lambda: v.integrateBatchDevice([d_cloud.data_ptr()], H, W, nf * 4, [pose]),
        "getFxn": lambda: v.getFxn(PTS),
        "getTSDFValue": lambda: v.getTSDFValue(PTS),
        "renderView": lambda: v.renderView(pose),
        "reconstruct": mc.reconstruct,
        "save": lambda: v.save(str(tmp_path / "v.vol")),
        "getVoxelCenters": v.getVoxelCenters,
        "getContainingVoxels": lambda: v.getContainingVoxels(PTS),
        "setContainingVoxelsData": lambda: v.setContainingVoxelsData(PTS, 0.0, 1.0),
        "export_shard": v.export_shard,
        "isEmpty": v.isEmpty,
    }
    for name, call in calls.items():
        _raises(ESTATE, call)

    v._cfg.pool_log2 = 18
    v._push()
    v.reset()
    _fuse(v)
    _assert_same_nodes(fresh.download_nodes(), v.download_nodes())


def test_refused_reset_keeps_the_volume():
    v = _volume()
    _fuse(v)
    nodes, fxn = v.download_nodes(), v.getFxn(PTS)
    v.setResolution(500, 500, 500)
    _raises(EINVAL, v.reset)
    _assert_same_nodes(nodes, v.download_nodes())
    after = v.getFxn(PTS)
    assert np.array_equal(fxn[0], after[0]) and np.array_equal(fxn[1].view(np.uint32), after[1].view(np.uint32))
