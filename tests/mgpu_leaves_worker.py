"""Worker for tests/test_leaves_mgpu.py (one process per GPU, launched by torch.distributed.run on a box with >= 2 GPUs).

Every rank fuses its shard of a 512^3 volume; the shards are gathered device to device into a full volume on rank 0
(b200tsdf_gather_volume), whose getVoxelCenters / getOccupiedVoxelIndices / isEmpty must equal the C++ restatement's on the
unsharded stream bit for bit, order included.  Enumerating a shard itself is refused (B200TSDF_ESTATE)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cpu_tsdf_b200 as pkg  # noqa: E402
from cpu_tsdf_b200 import synth  # noqa: E402
from tests import leaves  # noqa: E402
from tests.common import CFG_512, frames  # noqa: E402


def make(cfg, device, **kw):
    v = pkg.TSDFVolumeOctree(device=device, pool_log2=18, **kw)
    v.setResolution(cfg["xres"], cfg["yres"], cfg["zres"])
    v.setGridSize(cfg.get("xsize", 3.0), cfg.get("ysize", 3.0), cfg.get("zsize", 3.0))
    v.setCameraIntrinsics(525.0, 525.0, cfg["cx"], cfg["cy"])
    v.setIntegrateColor(True)
    v.reset()
    return v


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ids = [pkg.TSDFVolumeOctree.commUniqueId() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    shard = make(CFG_512, local, shard_rank=rank, shard_count=world)
    shard.commInit(ids[0], rank, world)
    fs = list(frames(synth.S1, 6, stride=8, color=True, noise_seed=31))
    for pose, cloud in fs:
        shard.integrateCloud(cloud, None, pose)
    shard.sync()
    try:
        shard.getOccupiedVoxelIndices()
        raise AssertionError("a shard enumerated its leaves")
    except pkg.B200Error as e:
        assert "(code -5)" in str(e) and "b200tsdf_gather_volume" in str(e)
    full = make(CFG_512, local) if rank == 0 else None
    if rank == 0:
        assert full.isEmpty()
    shard.gatherVolume(full, 0)
    if rank == 0:
        from oracle.leaves_py import LeavesOracleVolume
        o = LeavesOracleVolume(**CFG_512, integrate_color=1); o.reset()
        for pose, cloud in fs:
            o.integrate(cloud, pose)
        assert not full.isEmpty()
        C, L = o.levels()
        n_occ = 0
        for n in leaves.nlevels_sweep(C, L):
            a, b = o.voxel_centers(n), full.getVoxelCenters(n)
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), n
        a, b = o.occupied_voxel_indices(), full.getOccupiedVoxelIndices()
        assert np.array_equal(a, b) and len(a) > 1000
        n_occ = len(b)
        print(f"MGPU_LEAVES_OK world={world} occupied={n_occ}")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
