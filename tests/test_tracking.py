"""Tracking (DESIGN.md §3i) without a GPU, on the host emulation of track.cuh (tests/emu/track_emu.cpp).

* Per sample, r and g are the emulated query_point's mode-1 value and gradient at q, bit for bit (query_point is pinned to the
  reference by tests/test_queries.py); the inlier flag is exactly its definition.
* One iteration's A, b, sum rho r^2, sum r^2 and inlier count equal a float64 numpy statement of the same sums to 1e-12
  relative; solve6 and se3_exp_left equal numpy / scipy.
* On S1 (room + sphere) a held-out frame converges from perturbed poses to within the bounds below of the ground truth.
* On S2's wall view the smallest eigenvectors of the returned A are the motions the wall leaves free.
* Track-then-integrate over the noisy S1 orbit from the first ground-truth pose stays within the trajectory bounds below."""
import functools

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from cpu_tsdf_b200 import TRACK_CONVERGED, TrackParams, depth_to_cloud, synth
from tests.emu import track_py

CAM = synth.Camera()
# truncation 0.1 m: the basin of a point-to-SDF tracker is about the truncation band
VOL = dict(xsize=3.0, ysize=3.0, zsize=3.0, cx=CAM.cx, cy=CAM.cy, max_dist_pos=0.1, max_dist_neg=0.1, pool_log2=16)


@functools.lru_cache(maxsize=None)
def volume(res, color, scene="S1", step=10, noise=None, size=3.0):
    v = track_py.TrackEmuVolume(xres=res, yres=res, zres=res, integrate_color=int(color), **{**VOL, "xsize": size, "ysize": size, "zsize": size})
    v.reset()
    sc = getattr(synth, scene)
    for f in range(0, 100, step):
        pose = synth.orbit_pose(sc, f, 100)
        v.integrate(synth.make_frame(sc, pose, CAM, color=color, noise_seed=noise, frame=f), pose)
    return v


def perturb(pose, rot_deg, trans_m):
    d = np.eye(4)
    d[:3, :3] = Rotation.from_rotvec(np.radians(rot_deg)).as_matrix()
    d[:3, 3] = trans_m
    return d @ pose


def errors(pose, gt):
    return (float(np.linalg.norm(pose[:3, 3] - gt[:3, 3])),
            float(np.degrees(np.linalg.norm(Rotation.from_matrix(pose[:3, :3] @ gt[:3, :3].T).as_rotvec()))))


def held_out(f, scene=synth.S1, **kw):
    gt = synth.orbit_pose(scene, f, 100)
    return gt, synth.make_frame(scene, gt, CAM, **kw)


# ---- 1. per-sample values ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res,color", [(256, False), (256, True), (512, False), (512, True)])
def test_sample_residuals_are_the_query(res, color):
    v = volume(res, color)
    gt, frame = held_out(5, color=color, noise_seed=4, frame=5)
    pose = perturb(gt, [1.0, -0.5, 0.7], [0.01, 0.015, -0.02])
    for stride in (1, 3):
        s = v.samples(frame, pose, stride)
        u, vv = s["u"], s["v"]
        assert np.array_equal(s["finite"], np.isfinite(frame[vv, u, :3]).all(1))
        # q: (float) rows 0..2 of the pose applied as affine_mul_f, restated in numpy float32 without contraction
        m = pose[:3].astype(np.float32)
        x = frame[vv, u, :3]
        q = m[:, 3] + (m[:, 0] * x[:, :1] + (m[:, 1] * x[:, 1:2] + m[:, 2] * x[:, 2:3]))
        fin = s["finite"]
        assert np.array_equal(s["q"][fin].view(np.uint32), q[fin].view(np.uint32))
        val, grad, _, ok = v.query(s["q"][fin], what=3, mode=1)
        assert np.array_equal(ok, s["ok"][fin])
        assert np.array_equal(val[ok].view(np.uint32), s["r"][fin][ok].view(np.uint32))
        assert np.array_equal(grad[ok].view(np.uint32), s["g"][fin][ok].view(np.uint32))
        prm = TrackParams.default()
        want = s["ok"] & (s["wlo"] > prm.w_min) & (np.abs(s["r"]) < prm.d_max)
        assert np.array_equal(s["inlier"], want)
        assert 0.5 * fin.sum() < want.sum() < fin.sum(), (want.sum(), fin.sum())      # most points, not all


# ---- 2. normal equations -------------------------------------------------------------------------------------------------
def numpy_sums(s, prm):
    i = s["inlier"]
    q = s["q"][i].astype(np.float64); g = s["g"][i].astype(np.float64); r = s["r"][i].astype(np.float64)
    J = np.concatenate([np.cross(q, g), g], 1)
    rho = np.where(np.abs(r) <= prm.huber_delta, 1.0, prm.huber_delta / np.abs(r))
    A = (J * rho[:, None]).T @ J
    b = (J * (rho * r)[:, None]).sum(0)
    return A, b, float((rho * r * r).sum()), float((r * r).sum()), int(i.sum())


@pytest.mark.parametrize("res,color,stride", [(256, False, 1), (256, True, 2), (512, True, 4)])
def test_normal_equations_equal_float64_numpy(res, color, stride):
    v = volume(res, color)
    gt, frame = held_out(35, color=color, noise_seed=4, frame=35)
    pose = perturb(gt, [-1.5, 1.0, 0.5], [-0.02, 0.01, 0.02])
    prm = TrackParams.default(huber_delta=0.05)                  # so that both branches of the Huber weight are taken
    s = v.samples(frame, pose, stride)
    sums = v.sums(frame, pose, stride, prm)
    A, b, rr, r2, n = numpy_sums(s, prm)
    assert (np.abs(s["r"][s["inlier"]]) > prm.huber_delta).sum() > 100
    iu = np.triu_indices(6)
    got_A = np.zeros((6, 6)); got_A[iu] = sums[:21]; got_A = got_A + np.triu(got_A, 1).T
    assert sums[29] == n
    assert np.allclose(got_A, A, rtol=1e-12, atol=1e-12 * np.abs(A).max())
    assert np.allclose(sums[21:27], b, rtol=1e-12, atol=1e-12 * np.abs(b).max())
    assert abs(sums[27] - rr) <= 1e-12 * rr and abs(sums[28] - r2) <= 1e-12 * r2


def test_solve6_and_exp_equal_numpy_scipy():
    rng = np.random.default_rng(11)
    for _ in range(200):
        M = rng.standard_normal((6, 6)) * rng.uniform(0.1, 10, 6)
        A = M @ M.T + 1e-3 * np.eye(6)
        b = rng.standard_normal(6)
        lam = rng.choice([0.0, 1e-4, 0.1])
        x, ok = track_py.solve6(A, lam, b)
        assert ok
        want = np.linalg.solve(A + lam * np.diag(np.diag(A)), -b)
        assert np.allclose(x, want, rtol=1e-8, atol=1e-10 * np.abs(want).max())
    assert not track_py.solve6(-np.eye(6), 0.0, np.ones(6))[1]                 # a pivot <= 0
    assert not track_py.solve6(np.diag([1, 1, 1, 1, 1, 0.0]), 0.0, np.ones(6))[1]
    for k in range(200):
        T = np.eye(4)
        T[:3, :3] = Rotation.from_rotvec(rng.standard_normal(3)).as_matrix(); T[:3, 3] = rng.standard_normal(3)
        xi = rng.standard_normal(6) * (10.0 ** rng.uniform(-9, 0.4))
        E = np.eye(4)
        w, vel = xi[:3], xi[3:]
        th = np.linalg.norm(w)
        E[:3, :3] = Rotation.from_rotvec(w).as_matrix()
        W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        if th > 1e-6:
            V = np.eye(3) + (1 - np.cos(th)) / th**2 * W + (th - np.sin(th)) / th**3 * W @ W
        else:
            V = np.eye(3) + 0.5 * W + W @ W / 6
        E[:3, 3] = V @ vel
        got = track_py.se3_exp_left(xi, T)
        assert np.allclose(got, E @ T, atol=1e-12 * max(1.0, np.abs(T).max())), k
        assert np.abs(got[:3, :3] @ got[:3, :3].T - np.eye(3)).max() < 1e-15 * 8


# ---- 3. convergence on S1 ------------------------------------------------------------------------------------------------
# Bounds for the 256^3 / 3 m volume of ten S1 frames (truncation 0.1 m, voxels 11.7 mm), noise-free held-out frames, the
# default schedule.  Observed on the emulation: at most 2.6 mm and 0.10 deg over these eight starts.
S1_TRANS_BOUND, S1_ROT_BOUND = 0.005, 0.2
PERTURBATIONS = [([2.0, -1.5, 1.0], [0.03, -0.02, 0.025]), ([-3.0, 1.0, 2.0], [-0.04, 0.0, 0.02]),
                 ([0.0, 2.5, 0.0], [0.0, 0.03, -0.03]), ([1.0, 1.0, -2.0], [0.02, 0.02, 0.02])]


@pytest.mark.parametrize("f", [5, 45])
@pytest.mark.parametrize("k", range(len(PERTURBATIONS)))
def test_converges_on_s1(f, k):
    v = volume(256, False)
    gt, frame = held_out(f)
    rot, trans = PERTURBATIONS[k]
    pose, res = v.track(frame, perturb(gt, rot, trans))
    te, re = errors(pose, gt)
    assert res["status"] == TRACK_CONVERGED, res
    assert te < S1_TRANS_BOUND and re < S1_ROT_BOUND, (te, re)
    assert errors(perturb(gt, rot, trans), gt)[0] > 0.03                # the start is well outside the bounds
    assert len(res["log"]) == sum(res["iters"]) and res["inliers"] == res["log"][-1]["inliers"]


def test_uint16_depth_is_tracked_as_its_cloud():
    v = volume(256, False)
    gt, frame = held_out(25)
    z = frame[..., 2]
    d16 = np.where(np.isfinite(z), np.round(z * 1000), 0).astype(np.uint16)
    p0 = perturb(gt, [1.0, 1.0, 1.0], [0.02, -0.02, 0.02])
    a = v.track(d16, p0)
    b = v.track(depth_to_cloud(d16, v.intrinsics(), None, 1e-3), p0)
    assert np.array_equal(a[0], b[0]) and a[1]["status"] == b[1]["status"] == TRACK_CONVERGED
    assert np.array_equal(a[1]["A"], b[1]["A"])


# ---- 4. degeneracy on S2 -------------------------------------------------------------------------------------------------
def test_wall_view_reports_its_free_motions():
    """S2 frame 0 looks along +x at the wall x = R and sees nothing else: sliding along the wall (v_y, v_z) and turning about
    its normal (omega_x) change no residual, so the three smallest eigenvectors of A span exactly those three axes."""
    v = volume(256, False, "S2", size=5.0)                         # (S2's walls are 2 m from the centre)
    gt, frame = held_out(0, synth.S2)
    pose, res = v.track(frame, perturb(gt, [0.0, 0.5, 0.5], [0.02, 0.0, 0.0]))
    A = res["A"]
    w, V = np.linalg.eigh(A)
    free = V[:, :3]
    assert np.linalg.norm(free[[0, 4, 5]], axis=0).min() > 0.999, free
    assert w[2] < 1e-2 * w[3], w                                     # (observed: 1.4e-3)
    assert abs(pose[0, 3] - gt[0, 3]) < 0.005                        # the constrained direction is found


# ---- 5. closed loop ------------------------------------------------------------------------------------------------------
# Every second frame of the noisy S1 orbit, tracked from the previous estimate and then fused with it, from the first
# ground-truth pose: steps of 7.2 deg and 12.6 cm, 19 tracked frames.  Observed on the emulation: worst 27 mm and 1.11 deg.
LOOP_TRANS_BOUND, LOOP_ROT_BOUND = 0.04, 1.5


def test_track_then_integrate_loop():
    v = track_py.TrackEmuVolume(xres=256, yres=256, zres=256, **VOL)
    v.reset()
    prm = TrackParams.default(levels=2, stride=[4, 2], iters=[10, 6])
    est = synth.orbit_pose(synth.S1, 0, 100)
    v.integrate(synth.make_frame(synth.S1, est, CAM, noise_seed=9, frame=0), est)
    worst = (0.0, 0.0)
    for f in range(2, 40, 2):
        gt = synth.orbit_pose(synth.S1, f, 100)
        frame = synth.make_frame(synth.S1, gt, CAM, noise_seed=9, frame=f)
        est, res = v.track(frame, est, prm)
        assert res["status"] in (0, 1), res
        te, re = errors(est, gt)
        worst = (max(worst[0], te), max(worst[1], re))
        v.integrate(frame, est)
    assert worst[0] < LOOP_TRANS_BOUND and worst[1] < LOOP_ROT_BOUND, worst
