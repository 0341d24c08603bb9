"""Depth images without a GPU: the per-pixel routine of k_depth_unproject (depth.cuh) compiled for the host
(tests/emu/depth_emu.cpp) against the numpy statement of the contract, cpu_tsdf_b200.depth_to_cloud, byte for byte; and the
oracle fed depth_to_cloud clouds of synthetic frames, to show that the test inputs exercise fusion."""
import numpy as np
import pytest

from cpu_tsdf_b200 import depth_to_cloud, synth
from oracle.oracle_py import OracleVolume
from tests.common import CAM, CFG_256
from tests.emu import depth_py

INTR = (CAM.fx, CAM.fy, CAM.cx, CAM.cy)


def depth_frame(cloud):
    """the uint16 depth map (z in mm, NaN -> 0) and R, G, B image of a synthetic colour frame [H, W, 8]"""
    z = cloud[..., 2]
    depth = np.where(np.isfinite(z), np.clip(np.rint(z * 1000.0), 0, 65535), 0).astype(np.uint16)
    b = np.ascontiguousarray(cloud).view(np.uint8).reshape(cloud.shape[0], cloud.shape[1], 32)
    return depth, np.ascontiguousarray(b[..., [18, 17, 16]])


def every_u16():
    """a 256 x 256 map holding every uint16 value once"""
    return np.arange(65536, dtype=np.uint32).astype(np.uint16).reshape(256, 256)


def special_f32(h, w, seed=0):
    """float32 depths over the special values: +-0, denormals, FLT_MAX, +-inf, NaNs with payloads, negative and ordinary
    depths, spread over an h x w map"""
    rng = np.random.default_rng(seed)
    bits = np.array([0x00000000, 0x80000000, 0x00000001, 0x807fffff, 0x00400000, 0x7f7fffff, 0xff7fffff, 0x7f800000, 0xff800000,
                     0x7fc00000, 0x7fc00123, 0x7f800001, 0xffc00000, 0xffffffff, 0x3f800000, 0xbf800000], np.uint32)
    special = bits.view(np.float32)
    ordinary = rng.uniform(-5.0, 8.0, h * w).astype(np.float32)
    vals = np.where(rng.random(h * w) < 0.3, special[rng.integers(0, len(special), h * w)], ordinary)
    return np.ascontiguousarray(vals.reshape(h, w).astype(np.float32))


def rgb_of(h, w, seed=1):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def camera(w, h):
    """a w x h camera with an off-centre principal point"""
    f = 525.0 * w / 640
    return (f, f * 1.01, 0.47 * (w - 1) + 3.25, 0.53 * (h - 1) - 2.5)


def cases():
    """(name, depth, intrinsics, rgb, scale): the maps the CPU and the GPU tests both cover"""
    out = []
    u16 = every_u16()
    for scale in (1e-3, 2e-4, 1.0, 3e34):          # 3e34: every depth from 11343 up overflows to inf
        out.append((f"u16_all_{scale:g}", u16, INTR, None, scale))
    out.append(("u16_all_rgb", u16, INTR, rgb_of(256, 256), 1e-3))
    for w, h in ((640, 480), (643, 479)):
        rng = np.random.default_rng(w)
        d = rng.integers(0, 9000, (h, w)).astype(np.uint16)
        d[rng.random((h, w)) < 0.1] = 0
        out.append((f"u16_{w}x{h}", d, camera(w, h), None, 1e-3))
        out.append((f"u16_{w}x{h}_rgb", d, camera(w, h), rgb_of(h, w, w), 2e-4))
        out.append((f"f32_{w}x{h}", special_f32(h, w, w), camera(w, h), None, 1.0))
        out.append((f"f32_{w}x{h}_rgb_scaled", special_f32(h, w, w + 1), camera(w, h), rgb_of(h, w, h), 0.25))
    return out


CASES = cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_emulated_routine_equals_depth_to_cloud(case):
    _, depth, intr, rgb, scale = case
    want = depth_py.cloud_pixels(depth_to_cloud(depth, intr, rgb, scale))
    got = depth_py.depth_to_pixels(depth, intr, rgb, scale)
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=-1))[:5]


def test_contract_details():
    """the cases the contract names, stated directly on depth_to_cloud"""
    d = np.array([[0.0, -0.0, np.nan, np.inf, -np.inf, -2.0, 1.5, 3e38]], np.float32)
    c = depth_to_cloud(d, (500.0, 500.0, 1.0, 0.0), None, 2.0)
    bits = c.view(np.uint32)
    invalid = [0, 1, 2, 3, 4, 7]                   # 0, -0, NaN, +-inf and 3e38 * 2 = inf
    assert np.all(bits[0, invalid, :3] == 0x7fc00000)
    assert c[0, 5, 2] == -4.0 and c[0, 5, 0] == np.float32(-16.0 / 500.0)    # negative z passes through
    assert c[0, 6, 2] == 3.0
    assert np.all(c[..., 3] == 1.0) and np.all(bits[..., 4] == 0xff000000) and np.all(bits[..., 5:] == 0)
    rgb = np.array([[[10, 20, 30]] * 8], np.uint8)
    assert np.all(depth_to_cloud(d, (500.0, 500.0, 1.0, 0.0), rgb, 2.0).view(np.uint8)[0, :, 16:20] == [30, 20, 10, 255])


def test_oracle_fuses_depth_frames():
    """the oracle fed depth_to_cloud clouds of synthetic frames (depth = z in mm, NaN -> 0) builds a volume with surface"""
    o = OracleVolume(**CFG_256, integrate_color=1)
    o.reset()
    for f in range(3):
        pose = synth.orbit_pose(synth.S1, 4 * f, 100)
        depth, rgb = depth_frame(synth.make_frame(synth.S1, pose, CAM, color=True, noise_seed=3, frame=f))
        assert (depth > 0).mean() > 0.5
        o.integrate(depth_to_cloud(depth, INTR, rgb, 1e-3), pose)
    n = o.dump_nodes()
    dw = n["dw"].reshape(-1, 2)
    assert o.stats().n_add_observation > 10000 and len(n["keys"]) > 10000
    assert np.any(dw[:, 1] > 0) and np.any((dw[:, 0] > -1) & (dw[:, 0] < 1) & (dw[:, 1] > 0))
