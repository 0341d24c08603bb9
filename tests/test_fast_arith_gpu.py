"""The brick kernels' arithmetic shortcuts (cpu_tsdf_b200/csrc/obs_fast.cuh) on the H100, each against a plain float64
statement of the same operation, at the limits of the configurations that select them:

* div_recip / div_with, the five divisions of addObservation in k_bricks, against __fdiv_rn, and __fdiv_rn against the
  correctly rounded float32 (float64 (a) / float64 (b)): every mantissa of the divisor binades at both ends of each divisor
  range, numerators of every exponent, and random pairs over the operand box that Params::exact_div_ok admits;
* observe_issue's guarded projection and tsdf_core.cuh::project1 against trunc (float64 (x) fx / float64 (z) + c) with the
  x86 conversion, near every decision integer, on cameras up to the limits of fast_proj;
* float_at_least (device) and at_least (host) against the double comparisons they stand for.

The probe (tests/cuda/fast_arith_probe.cu) calls the headers' own functions with Params from derive_params."""
import ctypes as C
import zlib

import numpy as np
import pytest

from tests.test_fast_arith import load_probe, make_config, probe_params

pytestmark = pytest.mark.gpu

F32 = np.float32
NE = 278                                            # exponent buckets of the division map: 0 for +-0, ilogb (|x|) + 150 otherwise


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def f32(x):
    return float(F32(x))


# ---- division --------------------------------------------------------------------------------------------------------------
# The operand box of the brick kernels' divisions, for every configuration exact_div_ok admits
# (max_dist_neg in [1e-6f, 1e6f], |max_dist_pos| <= 1e6f, max_weight in [0, 1e9]):
#   d_new / max_dist_neg    divisor in [1e-6f, 1e6f], numerator in [-divisor, max_dist_pos] (d_new clamped);
#   sum / (w + 1)           divisor in [1, 1e9 + 1]; distance numerators d w + d_new with |d| <= 1e6f / 1e-6f, so |.| < 1.1e21;
#                           colour numerators w c + c' in [0, 255 (1e9 + 1)], 0 or >= min (max_weight, 1) >= 1e-20 (w is 0,
#                           max_weight or >= 1; c, c' are integers), divided by div_fast without the guard.
# The numerators are data (depth, pose, earlier frames), so their lower end is the subnormal range: d_new = z - vz is an exact
# difference of two floats, and with min_sensor_dist = 0 nothing keeps vz, and with it |d_new|, away from 2^-149.
DIV_BOXES = {                     # name: divisor range, |numerator| range, signed, negative side <= divisor, div_fast alone
    "d_new / max_dist_neg": ((f32(1e-6), f32(1e6)), (1e-45, f32(1e6)), True, True, False),
    "distance / (w + 1)": ((1.0, f32(1e9 + 1)), (1e-45, f32(1.1e21)), True, False, False),
    "colour / (w + 1)": ((1.0, f32(1e9 + 1)), (f32(1e-20), f32(255 * (1e9 + 1))), False, False, True),
}
# binades swept over every mantissa: the ends of both divisor ranges (1e-6f is in [2^-20, 2^-19), 1e6f in [2^19, 2^20),
# 1e9 + 1 in [2^29, 2^30)) and their neighbours
EXHAUSTIVE_BINADES = [-21, -20, -19, -1, 0, 1, 18, 19, 20, 28, 29, 30]


def ebucket(x):
    x = np.abs(np.asarray(x, F32))
    out = np.zeros(x.shape, np.int64)
    nz = x > 0
    out[nz] = np.floor(np.log2(x[nz].astype(np.float64))).astype(np.int64) + 150
    return out


def map_numerators():
    """a fixed set of numerators: eight mantissas of every exponent -149 ... 127, both signs, and +-0"""
    rng = np.random.default_rng(7)
    mant = np.concatenate([[1.0, 1.0 + 2.0 ** -23, 1.5, 2.0 - 2.0 ** -23], rng.uniform(1, 2, 4)])
    mag = np.unique(np.array([np.ldexp(m, e) for e in range(-149, 128) for m in mant], np.float64).astype(F32))
    mag = mag[(mag > 0) & np.isfinite(mag)]
    return np.concatenate([mag, -mag, np.array([0.0, -0.0], F32)]).astype(F32)


def div_map(binades, mstep, num, max_first=64):
    lib = load_probe()
    be = np.asarray(binades, np.int32)
    hist = np.zeros(NE * NE, np.uint64)
    n = C.c_ulonglong(0)
    first = np.zeros(4 * max_first, F32)
    assert lib.probe_div_map(len(be), ptr(be), mstep, len(num), ptr(num), ptr(hist), C.byref(n), ptr(first), max_first) == 0
    return hist.reshape(NE, NE), n.value, first[:4 * min(n.value, max_first)].reshape(-1, 4)


@pytest.fixture(scope="module")
def division_map():
    """mismatches of div_with against __fdiv_rn by (exponent of a, exponent of b): every mantissa of EXHAUSTIVE_BINADES, and
    every 97th mantissa of every binade 2^-28 ... 2^38 (the divisor ranges with 2^8 of margin on both sides)"""
    num = map_numerators()
    h1, n1, f1 = div_map(EXHAUSTIVE_BINADES, 1, num)
    h2, n2, f2 = div_map(list(range(-28, 39)), 97, num)
    return h1 + h2, n1 + n2, np.concatenate([f1, f2]), num


def describe(hist):
    """per divisor binade with mismatches: (log2 b, largest log2 |a| below 2^64 of a mismatching nonzero numerator (quotient or
    remainder subnormal), mismatches at a = +-0); the mismatches above are overflows of the quotient"""
    out = []
    for b in np.flatnonzero(hist.sum(axis=0)):
        a = np.flatnonzero(hist[1:150 + 64, b])
        out.append((int(b) - 150, int(a.max()) + 1 - 150 if len(a) else None, int(hist[0, b])))
    return out


# div_fast is trusted for a = +-0 and |a| >= 2^-64 (obs_fast.cuh DIV_FAST_MIN); div_with sends the rest to __fdiv_rn
DIV_FAST_MIN_LOG2 = -64


def test_division_map_is_clean_around_the_reachable_box(division_map):
    """div_fast has no mismatch anywhere in the box it is used on, widened by 2^8 on every side: divisors 2^-28 ... 2^38,
    numerators +-0 and 2^-72 <= |a| < 2^79 (the largest numerator is below 1.1e21 < 2^70)."""
    hist, n, first, num = division_map
    b_lo, b_hi = -28 + 150, 38 + 150
    a_lo, a_hi = DIV_FAST_MIN_LOG2 - 8 + 150, 70 + 8 + 150
    d = describe(hist)
    print(f"\ndivision map: {n} mismatching pairs of {len(num)} numerators x divisors of 12 whole and 67 sampled binades; "
          f"(log2 b, largest log2 |a| < 64 that mismatches, mismatches at +-0):", d, "first:", first[:4].tolist())
    assert hist[0, b_lo:b_hi + 1].sum() == 0, d
    assert hist[a_lo:a_hi + 1, b_lo:b_hi + 1].sum() == 0, d


def test_division_map_sees_every_numerator_exponent(division_map):
    """the map's numerators reach both exponent limits and both signed zeros (a map that skipped them would pass vacuously)"""
    num = division_map[3]
    b = ebucket(num)
    assert b.min() == 0 and set(range(1, 278)) <= set(b.tolist())
    z = num[num == 0].view(np.uint32)
    assert set(z.tolist()) == {0, 0x80000000}


@pytest.mark.parametrize("box", list(DIV_BOXES))
def test_div_with_matches_fdiv_rn_on_random_pairs(box):
    """4e8 random pairs per box (1.2e9 in all), the divisor's bits uniform over its range, the numerator's over its range
    (so every binade of |a| from 2^-149 up is sampled alike), +-0 one time in 64"""
    (b_lo, b_hi), (a_min, a_max), signed, neg_le_b, raw = DIV_BOXES[box]
    n = C.c_ulonglong(0)
    first = np.zeros(4 * 16, F32)
    rc = load_probe().probe_div_random(1234 + len(box), 400_000_000, b_lo, b_hi, a_min, a_max, int(signed), int(neg_le_b), int(raw),
                                       C.byref(n), ptr(first), 16)
    assert rc == 0
    assert n.value == 0, first[:4 * min(n.value, 16)].reshape(-1, 4).tolist()


def near_midpoint_pairs(n_b, rng):
    """(a, b) whose exact quotient lies within t 2^-24 ulp of a rounding midpoint (t odd, |t| < 64): b = B 2^-23 and the
    midpoint m = M 2^-24 (B, M odd) with B M = t mod 2^25, so a = (B M - t) 2^-47 is a float and a / b = m - t 2^-47 / b.
    Random operands almost never come this close; a quotient sequence without its Newton step rounds some of them wrong."""
    B = rng.integers(2 ** 22, 2 ** 23, n_b, dtype=np.uint64) * 2 + 1
    inv = B.copy()
    for _ in range(6):                                     # inverse of B modulo 2^64 (Newton's iteration, odd B)
        inv = inv * (np.uint64(2) - B * inv)
    t = np.concatenate([np.arange(1, 64, 2), -np.arange(1, 64, 2)]).astype(np.int64)
    M = ((t[None, :].astype(np.uint64) * inv[:, None]) & np.uint64(2 ** 25 - 1)).astype(np.int64)
    Bm = np.broadcast_to(B[:, None].astype(np.int64), M.shape)
    ok = M > 2 ** 24                                       # m in (1, 2)
    num = Bm[ok] * M[ok] - np.broadcast_to(t, M.shape)[ok]
    a = np.ldexp(num.astype(np.float64), -47)
    b = np.ldexp(Bm[ok].astype(np.float64), -23)
    assert np.array_equal(a.astype(F32).astype(np.float64), a)
    # into the divisor ranges: b scaled by 2^-20 ... 2^28, a by the same and by a random power of two, random signs
    e_b = rng.integers(-20, 29, len(a))
    e_a = e_b + rng.integers(-40, 40, len(a))
    sign = np.where(rng.integers(0, 2, len(a)) == 1, -1.0, 1.0)
    return (sign * np.ldexp(a, e_a)).astype(F32), np.ldexp(b, e_b).astype(F32)


def test_division_near_midpoints():
    """div_with and __fdiv_rn against the correctly rounded quotient on 6e5 pairs whose quotient is within 2^-18 ulp of a
    rounding midpoint"""
    a, b = near_midpoint_pairs(20_000, np.random.default_rng(3))
    n = len(a)
    ow, oe = np.empty(n, F32), np.empty(n, F32)
    assert load_probe().probe_div(n, ptr(a), ptr(b), ptr(ow), ptr(oe)) == 0
    ref = (a.astype(np.float64) / b.astype(np.float64)).astype(F32)
    for got in (oe, ow):
        bad = got.view(np.uint32) != ref.view(np.uint32)
        assert not bad.any(), (int(bad.sum()), list(zip(a[bad][:3], b[bad][:3], got[bad][:3], ref[bad][:3])))
    assert n > 500_000


def test_fdiv_rn_is_correctly_rounded():
    """__fdiv_rn (and div_with) against float32 (float64 (a) / float64 (b)), which is correctly rounded (53 >= 2 * 24 + 2),
    on 1.6e7 pairs: numerators of every finite magnitude and both signed zeros, divisors over both divisor ranges"""
    rng = np.random.default_rng(11)
    n = 16_000_000
    a = rng.integers(0, 0x7F800000, n, dtype=np.uint32)
    a[rng.integers(0, 64, n) == 0] = 0
    a |= rng.integers(0, 2, n, dtype=np.uint32) << 31
    a = a.view(F32)
    lo, hi = F32(1e-6).view(np.uint32), F32(1e9 + 1).view(np.uint32)
    b = rng.integers(lo, hi + 1, n, dtype=np.uint32).view(F32)
    ow, oe = np.empty(n, F32), np.empty(n, F32)
    assert load_probe().probe_div(n, ptr(a), ptr(b), ptr(ow), ptr(oe)) == 0
    with np.errstate(over="ignore"):
        ref = (a.astype(np.float64) / b.astype(np.float64)).astype(F32)
    bad = oe.view(np.uint32) != ref.view(np.uint32)
    assert not bad.any(), list(zip(a[bad][:5], b[bad][:5], oe[bad][:5], ref[bad][:5]))
    assert ((a == 0) & (np.signbit(a))).sum() > 10_000 and (np.abs(a) < F32(2.0 ** -126)).sum() > 10_000
    # div_with agrees for every numerator below 2^79 (the brick kernels' numerators stay below 2^70)
    badw = (np.abs(a) < F32(2.0 ** 79)) & (ow.view(np.uint32) != ref.view(np.uint32))
    assert not badw.any(), list(zip(a[badw][:5], b[badw][:5], ow[badw][:5], ref[badw][:5]))


# ---- projection ------------------------------------------------------------------------------------------------------------
CAMS = {                                            # (fx, fy, cx, cy, width, height)
    "default": (525.0, 525.0, 319.5, 239.5, 640, 480),
    "tum": (517.3, 516.5, 318.6, 255.3, 640, 480),
    "strip8191": (4096.0, 128.0, 4095.5, 31.5, 8191, 64),      # the widest image with fast_proj on
    "c_edge": (525.0, 525.0, 9999.5, -9999.5, 640, 480),      # the edge of the |c| < 1e4 gate
    "fx1": (1.0, 1.0, 319.5, 239.5, 640, 480),
    "fx1e5": (1e5, 1e5, 319.5, 239.5, 640, 480),
    "g6_8192": (4096.0, 128.0, 4095.5, 31.5, 8192, 64),       # fast_proj off: the double expression answers
}


def cam_config(cam, **kw):
    fx, fy, cx, cy, w, h = CAMS[cam]
    return dict(fx=fx, fy=fy, cx=cx, cy=cy, image_width=w, image_height=h, **kw)


def to_int_x86(a):
    """(int) of a double the way cvttsd2si does it: truncation toward zero, INT_MIN out of range or NaN"""
    ok = (a > -2147483649.0) & (a < 2147483648.0)
    out = np.full(a.shape, np.iinfo(np.int32).min, np.int64)
    out[ok] = np.trunc(a[ok]).astype(np.int64)
    return out


def depths(lo, hi, rng):
    """the sensor bounds and their float neighbours, powers of two in between +-1 ulp, a log-uniform sample"""
    z = [lo, hi, np.nextafter(F32(lo), F32(0)), np.nextafter(F32(lo), F32(np.inf)), np.nextafter(F32(hi), F32(0)),
         np.nextafter(F32(hi), F32(np.inf))]
    for e in range(int(np.floor(np.log2(lo))), int(np.ceil(np.log2(hi))) + 1):
        p = F32(2.0 ** e)
        z += [p, np.nextafter(p, F32(0)), np.nextafter(p, F32(np.inf))]
    z += list(np.exp(rng.uniform(np.log(lo), np.log(hi), 12)))
    z = np.array(z, F32)
    return np.unique(z[z > 0])


def decision_ints(n, rng):
    """-1 and 1 ... n; for wide axes both ends and 512 random integers"""
    if n <= 1024:
        return np.concatenate([[-1], np.arange(1, n + 1)])
    return np.unique(np.concatenate([[-1], np.arange(1, 33), np.arange(n - 31, n + 1), rng.integers(1, n + 1, 512)]))


def ladder(k, guard):
    """offsets around each decision integer k: 0, +-1 ... 4 ulps of float32 (k), +-{0.5, 0.99, 1.01, 2} guard"""
    sp = np.spacing(np.abs(k).astype(F32)).astype(np.float64)
    steps = [np.zeros_like(sp)] + [s * j * sp for j in (1, 2, 3, 4) for s in (1, -1)] + \
            [np.full_like(sp, s * m * guard) for m in (0.5, 0.99, 1.01, 2.0) for s in (1, -1)]
    return np.stack([k + d for d in steps], axis=1).ravel()


def observe_inputs(cam, guard, lo, hi, rng):
    """(vx, vy, vz) whose pixel coordinate along one axis sits on the ladder around a decision integer, the other axis at a
    random place in (or just outside) the image; vx, vy rounded to float32 and the reference recomputed from them"""
    fx, fy, cx, cy, w, h = CAMS[cam]
    out = []
    for axis, (n_axis, n_other) in enumerate(((w, h), (h, w))):
        t = ladder(decision_ints(n_axis, rng).astype(np.float64), guard)
        for z in depths(lo, hi, rng):
            other = rng.uniform(-2, n_other + 2, len(t))
            tu, tv = (t, other) if axis == 0 else (other, t)
            zd = np.float64(z)
            vx = ((tu - cx) * zd / fx).astype(F32)
            vy = ((tv - cy) * zd / fy).astype(F32)
            out.append((vx, vy, np.full(len(t), z, F32), np.full(len(t), axis)))
    return [np.concatenate(c) for c in zip(*out)]


@pytest.mark.parametrize("sensor", ["default", "min0"])
@pytest.mark.parametrize("cam", list(CAMS))
def test_observe_projection_matches_double(cam, sensor):
    """observe_issue<false> (u, v, in image) equals the reference's double expression for every input, and the float estimate's
    measured error stays within proj_guard / 1.5 (the error model behind the guard, on the hardware's rcp.approx)"""
    lo, hi = (0.3, 3.0) if sensor == "default" else (0.0, 3.0)
    cfg = cam_config(cam, min_sensor_dist=lo, max_sensor_dist=hi)
    p = probe_params(cfg)
    guard = p["proj_guard"]
    assert p["fast_proj"] == (0 if cam == "g6_8192" else 1)
    rng = np.random.default_rng(zlib.crc32(f"{cam}/{sensor}".encode()))
    vx, vy, vz, axis = observe_inputs(cam, guard, 0.3 if sensor == "default" else 1e-30, hi, rng)
    n = len(vz)
    u, v, inimg = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32)
    au, av = np.empty(n, F32), np.empty(n, F32)
    assert load_probe().probe_observe(C.byref(make_config(**cfg)), n, ptr(vx), ptr(vy), ptr(vz), ptr(u), ptr(v), ptr(inimg),
                                      ptr(au), ptr(av)) == 0
    fx, fy, cx, cy, w, h = CAMS[cam]
    zd = vz.astype(np.float64)
    a_ref = vx.astype(np.float64) * fx / zd + cx
    b_ref = vy.astype(np.float64) * fy / zd + cy
    u_ref, v_ref = to_int_x86(a_ref), to_int_x86(b_ref)
    in_ref = (vz >= F32(lo)) & (vz <= F32(hi)) & (vz > 0) & (u_ref >= 0) & (u_ref < w) & (v_ref >= 0) & (v_ref < h)
    assert np.array_equal(inimg.astype(bool), in_ref), np.flatnonzero(inimg.astype(bool) != in_ref)[:5]
    assert np.array_equal(u[in_ref], u_ref[in_ref]) and np.array_equal(v[in_ref], v_ref[in_ref])
    assert in_ref.mean() > 0.5
    if not p["fast_proj"]:
        return
    # the estimate's error, where the error model applies (the node is inside the sensor bounds)
    ok = (vz >= F32(lo)) & (vz <= F32(hi))
    err = np.maximum(np.abs(au[ok] - a_ref[ok]), np.abs(av[ok] - b_ref[ok]))
    print(f"\n{cam}/{sensor}: {n} inputs, proj_guard {guard:.3e}, max |estimate - double| {err.max():.3e} "
          f"= {err.max() / guard:.3f} proj_guard")
    assert err.max() <= guard / 1.5
    # the inputs straddle the guard band: inside it and just outside it, above and below integers
    t = np.where(axis == 0, a_ref, b_ref)[ok]
    d = t - np.round(t)
    inside, outside = np.abs(d) <= guard, (np.abs(d) > guard) & (np.abs(d) <= 2.5 * guard)
    for sel in (inside, outside):
        assert sel.mean() >= 0.2 and (sel & (d > 0)).mean() >= 0.05 and (sel & (d < 0)).mean() >= 0.05


P1_CAMS = {                                          # (f, c) along one axis
    "default": (525.0, 319.5), "c+edge": (525.0, 9999.5), "c-edge": (525.0, -9999.5), "f1": (1.0, 319.5),
    "f1e5": (1e5, 319.5), "f1e5_c-edge": (1e5, -9999.5),
}


@pytest.mark.parametrize("cam", list(P1_CAMS))
def test_project1_matches_double(cam):
    """tsdf_core.cuh::project1 (the general kernel's projection) equals trunc (float64 (x) f / float64 (z) + c) for every input
    near integers up to 3e4, and its float estimate's measured error stays below the 0.01 margin it accepts with"""
    f, c = P1_CAMS[cam]
    rng = np.random.default_rng(5)
    k = np.unique(np.concatenate([np.arange(-1, 70), rng.integers(1, 30000, 1500), np.arange(29950, 30001)])).astype(np.float64)
    steps = [0.0, 1e-3, 5e-3, 9.9e-3, 1.01e-2, 2e-2, 0.5]
    d = np.concatenate([[s * m for s in steps for m in (1, -1)], rng.uniform(-0.02, 0.02, 16)])
    t = (k[:, None] + d[None, :]).ravel()
    outs = []
    for axis, cfg in enumerate((dict(fx=f, cx=c), dict(fy=f, cy=c))):
        for z in depths(1e-3, 3.0, rng):
            x = ((t - c) * np.float64(z) / f).astype(F32)
            zz = np.full(len(t), z, F32)
            n = len(t)
            out, est = np.empty(n, np.int32), np.empty(n, F32)
            assert load_probe().probe_project1(C.byref(make_config(**cfg)), axis, n, ptr(x), ptr(zz), ptr(out), ptr(est)) == 0
            ref = x.astype(np.float64) * f / zz.astype(np.float64) + c
            want = to_int_x86(ref)
            assert np.array_equal(out, want), (axis, z, np.flatnonzero(out != want)[:5])
            outs.append(np.abs(est.astype(np.float64) - ref)[(ref > 0) & (ref < 3e4)])
    err = np.concatenate(outs).max()
    print(f"\nproject1 {cam}: max |estimate - double| {err:.3e} = {err / 0.01:.3f} of the 0.01 margin")
    assert err < 0.01


# ---- thresholds ------------------------------------------------------------------------------------------------------------
THRESH_PARAMS = [dict(), dict(max_dist_pos=0.05, max_dist_neg=0.02), dict(max_dist_neg=f32(1e-6), max_dist_pos=f32(1e6)),
                 dict(max_dist_neg=f32(1e6)), dict(max_dist_pos=-0.0), dict(max_dist_pos=1 / 32, max_dist_neg=1 / 32)]
GRIDS = [(3.0, 512), (3.0, 256), (10.0, 2048), (10.0, 4096), (4.0, 256)]


def test_float_thresholds_decide_like_the_double_ones():
    """for every rc threshold and every near threshold of the grids above, and every float d within 64 ulps of it:
    d < float_at_least (t) on the device, and d < at_least (t) on the host, equal (double) d < t"""
    lib = load_probe()
    ts, host_rc = [], []
    for prm in THRESH_PARAMS:
        p = probe_params(prm)
        ts += [-0.99, p["rc_thresh"]]
        host_rc += [p["rc_lo_f"], p["rc_hi_f"]]
    sizes = np.array([s / 2 ** l for s, res in GRIDS for l in range(int(np.log2(res)) + 1)], F32)
    nd, nh = np.empty(len(sizes)), np.empty(len(sizes))
    assert lib.probe_near_threshold(len(sizes), ptr(sizes), ptr(nd), ptr(nh)) == 0
    assert np.array_equal(nd, nh)
    t = np.array(ts + nd.tolist(), np.float64)
    dev, host = np.empty(len(t), F32), np.empty(len(t), F32)
    assert lib.probe_at_least(len(t), ptr(t), ptr(dev), ptr(host)) == 0
    assert np.array_equal(dev.view(np.uint32), host.view(np.uint32))
    assert np.array_equal(np.array(host_rc, F32).view(np.uint32), host[:len(host_rc)].view(np.uint32))
    for i in range(len(t)):
        d = around(F32(t[i]), 64)
        assert np.array_equal(d < dev[i], d.astype(np.float64) < t[i]), (t[i], dev[i])


def around(x, n):
    """the 2n + 1 floats centred on x, in order of value"""
    lo, hi = [x], [x]
    for _ in range(n):
        lo.append(np.nextafter(lo[-1], F32(-np.inf)))
        hi.append(np.nextafter(hi[-1], F32(np.inf)))
    return np.array(lo[::-1] + hi[1:], F32)
