"""The test-only probe of the brick kernels' arithmetic (tests/cuda/fast_arith_probe.cu): it builds for sm_90a with the engine's
own nvcc flags, and its host side derives Params the way the engine does.  The device checks are in test_fast_arith_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np

from cpu_tsdf_b200 import Config
from cpu_tsdf_b200.build import NVCC_FLAGS, nvcc_path

_lib = None


class ProbeParams(C.Structure):
    _fields_ = [("fast_proj", C.c_int32), ("exact_div_ok", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("L", C.c_int32), ("proj_guard", C.c_float), ("rc_lo_f", C.c_float), ("rc_hi_f", C.c_float),
                ("rc_thresh", C.c_double)]


def load_probe():
    """libfast_arith_probe.so, rebuilt when it is older than its sources"""
    global _lib
    if _lib is None:
        from tests.cuda.build_probe import build_probe
        lib = C.CDLL(build_probe())
        vp, i, f, u64 = C.c_void_p, C.c_int, C.c_float, C.c_ulonglong
        lib.probe_params.argtypes = [C.POINTER(Config), C.POINTER(ProbeParams)]
        lib.probe_div.argtypes = [i, vp, vp, vp, vp]
        lib.probe_div_map.argtypes = [i, vp, i, i, vp, vp, vp, vp, i]
        lib.probe_div_random.argtypes = [u64, C.c_longlong, f, f, f, f, i, i, i, vp, vp, i]
        lib.probe_observe.argtypes = [C.POINTER(Config), i, vp, vp, vp, vp, vp, vp, vp, vp]
        lib.probe_project1.argtypes = [C.POINTER(Config), i, i, vp, vp, vp, vp]
        lib.probe_at_least.argtypes = [i, vp, vp, vp]
        lib.probe_near_threshold.argtypes = [i, vp, vp, vp]
        _lib = lib
    return _lib


def make_config(**kw):
    """a b200tsdf_config with the engine's defaults (params_setup.h default_config) and the fields in `kw`"""
    c = Config()
    d = dict(xres=512, yres=512, zres=512, xsize=3.0, ysize=3.0, zsize=3.0, max_dist_pos=0.03, max_dist_neg=0.03, max_weight=100,
             min_sensor_dist=0.3, max_sensor_dist=3.0, fx=525.0, fy=525.0, cx=320.0, cy=240.0, image_width=640, image_height=480,
             max_cell_x=0.5, max_cell_y=0.5, max_cell_z=0.5, pool_log2=20, shard_rank=0, shard_count=1)
    d.update(kw)
    for k, v in d.items():
        setattr(c, k, v)
    for k in range(4):
        c.global_transform[5 * k] = 1.0
    return c


def probe_params(cfg: dict):
    """fast_proj, exact_div_ok, proj_guard, ... as derive_params sets them for the configuration `cfg` (host code only)"""
    out = ProbeParams()
    assert load_probe().probe_params(C.byref(make_config(**cfg)), C.byref(out)) == 0, cfg
    return {k: getattr(out, k) for k, _ in ProbeParams._fields_}


def test_probe_builds_for_sm90a(tmp_path):
    from tests.cuda.build_probe import build_probe
    assert "-fmad=false" in NVCC_FLAGS and "arch=compute_90a,code=sm_90a" in NVCC_FLAGS
    so = build_probe(force=True, out=str(tmp_path / "probe.so"))
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    elf = subprocess.run([cuobjdump, "--list-elf", so], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in elf
    sass = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True, check=True).stdout
    assert "MUFU.RCP" in sass and "k_div_map" in sass and "k_observe" in sass


def test_probe_params_match_the_engines_gates():
    """the regimes test_fast_arith_gpu.py relies on, as derive_params decides them"""
    p = probe_params({})
    assert p["fast_proj"] == 1 and p["exact_div_ok"] == 1 and 0 < p["proj_guard"] < 1e-3
    assert probe_params(dict(image_width=8192, image_height=64, fx=4096.0, cx=4095.5))["fast_proj"] == 0
    assert probe_params(dict(image_width=8191, image_height=64, fx=4096.0, cx=4095.5))["fast_proj"] == 1
    assert probe_params(dict(cx=9999.5, cy=-9999.5))["fast_proj"] == 1
    assert probe_params(dict(cx=10000.0))["fast_proj"] == 0
    f32 = lambda x: float(np.float32(x))
    assert probe_params(dict(max_dist_neg=f32(1e-6), max_dist_pos=f32(1e6)))["exact_div_ok"] == 1
    assert probe_params(dict(max_dist_neg=f32(1e6), max_weight=1e9))["exact_div_ok"] == 1
    assert probe_params(dict(max_dist_neg=1.2e-38))["exact_div_ok"] == 0
    assert probe_params(dict(max_weight=2e9))["exact_div_ok"] == 0
    # colour numerators w c + c' are divided without the tiny-numerator guard: w must be 0 or at least min (max_weight, 1)
    assert probe_params(dict(max_weight=0.0))["exact_div_ok"] == 1
    assert probe_params(dict(max_weight=1e-20))["exact_div_ok"] == 1
    assert probe_params(dict(max_weight=1e-30))["exact_div_ok"] == 0
