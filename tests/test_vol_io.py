"""The .vol writer's and parser's per-record routines (vol_io.cuh) on the host emulation (tests/emu/vol_emu.cpp), against
the reference's save (the C++ restatement of oracle/), on grid shapes and on the pin cases K1-K6 and E1-E5: the emitted, keyed, sorted and formatted body equals the reference's
bytes; the parser accepts those files and places every record where the reference's loader would; and it refuses (so the
engine falls back to its host loader) truncated bodies, nchild = 3, a tree shallower than the coarse depth or deeper than the
resolution, and a centre moved by one ulp, while trailing bytes after a valid body are accepted with the same volume."""
import struct

import numpy as np
import pytest

from cpu_tsdf_b200 import synth
from oracle.oracle_py import OracleVolume
from tests import dynamic_cases, general_cases
from tests.common import CAM, CFG_256, CFG_512, assert_same_nodes, frames
from tests.emu.vol_py import EmuVolVolume

SHAPES = [("256_rgb", CFG_256, 1), ("512", CFG_512, 0),
          ("128_c0.5", dict(xres=128, yres=128, zres=128, cx=CAM.cx, cy=CAM.cy, max_cell_x=0.5, max_cell_y=0.5, max_cell_z=0.5), 0),
          ("256_2.7_c0.3", dict(xres=256, yres=256, zres=256, xsize=2.7, ysize=2.7, zsize=2.7, cx=CAM.cx, cy=CAM.cy,
                                max_cell_x=0.3, max_cell_y=0.3, max_cell_z=0.3), 0)]


def split_file(raw):
    off = raw.index(b"#OCTREEBINARY\n") + len(b"#OCTREEBINARY\n") + 36
    return raw[:off], raw[off:]


def fused(cfg, color, tmp_path, nframes=3):
    kw = dict(cfg, track_variance=1, integrate_color=color)
    e = EmuVolVolume(**kw); e.reset()
    o = OracleVolume(**cfg, **({"integrate_color": 1} if color else {})); o.reset()
    scene = synth.S1 if cfg.get("xsize", 3.0) == 3.0 and "max_cell_x" not in cfg else synth.Scene(room_half=1.2, cam_radius=0.8)
    for pose, cloud in frames(scene, nframes, stride=7, color=bool(color), noise_seed=5):
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    p = tmp_path / "o.vol"
    assert o.save(str(p)) == 0
    return e, o, p.read_bytes()


@pytest.mark.parametrize("name,cfg,color", SHAPES, ids=[s[0] for s in SHAPES])
def test_body_and_parse_equal_the_reference(tmp_path, name, cfg, color):
    e, o, raw = fused(cfg, color, tmp_path)
    _, body = split_file(raw)
    assert e.body() == body
    fresh = EmuVolVolume(**dict(cfg, track_variance=1, integrate_color=color)); fresh.reset()
    st, n, ood = fresh.parse(body, bool(color))
    assert st == 1 and n * (43 if color else 40) == len(body) and ood == 0
    assert_same_nodes(o.dump_nodes(), fresh.dump_nodes(), rgb=bool(color), var=True)


# the dynamic scenes (pruning and re-splitting) and the exact-tie cases; K3 is RGBNormalized, a payload the emulation does not keep
PIN_CASES = [dynamic_cases.CASES[k] for k in ("K1", "K2", "K4", "K5", "K6")] + \
            [general_cases.CASES[k] for k in ("E1", "E2", "E3", "E4", "E5")]


@pytest.mark.parametrize("case", PIN_CASES, ids=[c.id for c in PIN_CASES])
def test_pin_cases(tmp_path, case):
    pool = {256: 17, 512: 18, 2048: 18, 4096: 19}[case.res]
    e = EmuVolVolume(**case.config(), track_variance=1, pool_log2=pool); e.reset()
    o = OracleVolume(**case.config()); o.reset()
    for pose, cloud in case.frames():
        o.integrate(cloud, pose); e.integrate(cloud, pose)
    p = tmp_path / "o.vol"
    assert o.save(str(p)) == 0
    _, body = split_file(p.read_bytes())
    assert e.body() == body
    fresh = EmuVolVolume(**case.config(), track_variance=1, pool_log2=pool); fresh.reset()
    st, n, _ = fresh.parse(body, bool(case.color))
    assert st == 1 and n * (43 if case.color else 40) == len(body)
    assert_same_nodes(o.dump_nodes(), fresh.dump_nodes(), rgb=bool(case.color), var=True)


def test_parser_refusals(tmp_path):
    e, o, raw = fused(CFG_256, 0, tmp_path, nframes=2)
    _, body = split_file(raw)
    R, n = 40, len(body) // 40
    sizes = [struct.unpack_from("<f", body, i * R + 20)[0] for i in range(n)]
    finest = int(np.argmin(sizes))

    def patched(i, at, fmt, val):
        b = bytearray(body); struct.pack_into(fmt, b, i * R + at, val); return bytes(b)

    cx = struct.unpack_from("<f", body, finest * R + 8)[0]
    refused = {
        "truncated": body[:-20],
        "nchild3": patched(5, 32, "<Q", 3),
        "shallow": patched(0, 32, "<Q", 0),
        "deep": patched(finest, 32, "<Q", 8),
        "ulp": patched(finest, 8, "<f", float(np.nextafter(np.float32(cx), np.float32(np.inf)))),
    }
    for name, b in refused.items():
        v = EmuVolVolume(**dict(CFG_256, track_variance=1)); v.reset()
        before = v.dump_nodes()
        st, _, _ = v.parse(b, False)
        assert st == 0, name
        after = v.dump_nodes()
        assert np.array_equal(before["keys"], after["keys"]) and np.array_equal(before["dw"], after["dw"]), name
    v = EmuVolVolume(**dict(CFG_256, track_variance=1)); v.reset()
    st, m, _ = v.parse(body + b"\x01" * 57, False)
    assert st == 1 and m == n
    assert_same_nodes(o.dump_nodes(), v.dump_nodes(), var=True)
    # a stored {d, w} that fusion does not produce is counted for the route check
    v = EmuVolVolume(**dict(CFG_256, track_variance=1)); v.reset()
    assert v.parse(patched(n - 1, 4, "<f", -0.5), False)[2] == 1
