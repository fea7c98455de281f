"""Rolling-shutter board poses (icc_set_pose_rolling_shutter, --pose_shutter rolling): each view's pose at its frame timestamp from corners
exposed row by row, with the views' velocities taken from their neighbours in time.

CPU part: the product's rolling-shutter header compiled for the CPU has the stated Jacobians and velocities; on a synthetic sequence with a
physical rolling shutter (tests/rolling_shutter_support.py) the oracle's rolling-shutter poses are closer to the truth at the frame time
than its global-shutter poses, its velocities match the truth, and the IMU-to-camera time offset from them is that of the true poses; a
zero line delay, a motionless camera and views without neighbours give back the global-shutter result; the library and the CLIs check
their arguments.
GPU part (-m gpu): the CUDA path reproduces the oracle for every camera model and both residuals, also for icc_optimize_board_points and at
full size (3000 views x 144 corners, with the wall time of global against rolling shutter), and the tool chain pose CLI -> rotation CLI
-> hot CLI runs with --pose_shutter rolling."""
import json
import os
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_models import CASES
from test_pose_estimation import _qdiff
from rolling_shutter_support import (FPS, H, LINE_DELAY, W, RsPoseOracle, product_rs_residual, product_rs_transform, product_rs_velocity,
                                     rs_sequence, view_velocities)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")
POSE_CLI = os.path.join(BIN, "estimate_camera_poses_from_checkerboard")
ROT_CLI = os.path.join(BIN, "estimate_imu_to_camera_rotation")
HOT_CLI = os.path.join(BIN, "continuous_time_imu_to_camera_calibration")
MODELS = [CASES[0], CASES[4]]
MODEL_IDS = [cm.MODEL_NAMES[m] for m, _ in MODELS]
ALL_IDS = [cm.MODEL_NAMES[m] for m, _ in CASES]


def _rot_err(q, q_true):
    return 2 * np.arccos(np.clip(np.abs(np.sum(q * q_true, 1)), 0, 1))


def _setup(api, model, k, board, mode="normalized"):
    api.set_camera(model, k, W, H); api.set_board_points(board); api.set_pose_error(mode)
    return api


def _poses(api, s, line_delay=LINE_DELAY):
    api.set_pose_rolling_shutter(line_delay, s["frame_t"])
    return api.estimate_board_poses(s["off"], s["ids"], s["uv"])


# ---- 1. the product's math on the CPU ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tangent", [0, 1], ids=["normalized", "tangent"])
def test_rs_residual_jacobians_match_central_differences(tangent):
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3 + tangent)
    for _ in range(30):
        q = Rotation.from_rotvec(rng.normal(0, 0.5, 3)).as_quat(); R = Rotation.from_quat(q).as_matrix()
        X = rng.normal(0, 0.1, 3); t = np.array([0.0, 0.0, 0.5]) - R @ X + rng.normal(0, 0.05, 3)
        wu = np.r_[rng.normal(0, 3, 3), rng.normal(0, 0.8, 3)]; tau = rng.uniform(0, 1 / FPS)
        P = R @ X + t
        meas = P / np.linalg.norm(P) + rng.normal(0, 0.02, 3) if tangent else P[:2] / P[2] + rng.normal(0, 0.02, 2)
        if tangent:
            meas = meas / np.linalg.norm(meas)
        r, front, J = product_rs_residual(tangent, meas, q, X, t, wu, tau)
        assert front
        h = 1e-6
        for j in range(6):
            d = np.zeros(6); d[j] = h
            def at(s):
                Rq = Rotation.from_matrix(R @ Rotation.from_rotvec(s * d[:3]).as_matrix()).as_quat()
                return product_rs_residual(tangent, meas, Rq, X, t + s * d[3:], wu, tau)[0]
            assert np.abs((at(1) - at(-1)) / (2 * h) - J[:, j]).max() < 1e-6 * max(1.0, np.abs(J).max())
        # the transform: exp(-tau [w]x)(P0 - tau u), the identity at tau = 0 and for w = u = 0
        A = Rotation.from_rotvec(-tau * wu[:3]).as_matrix()
        assert np.abs(product_rs_transform(P, wu, tau) - A @ (P - tau * wu[3:])).max() < 1e-14
        assert np.array_equal(product_rs_transform(P, wu, 0.0), P) and np.array_equal(product_rs_transform(P, np.zeros(6), tau), P)


def test_rs_velocity_formula():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(5)
    for _ in range(20):
        q = Rotation.from_rotvec(rng.normal(0, 1, (3, 3))).as_quat(); p = rng.normal(0, 1, (3, 3)); t = np.sort(rng.uniform(0, 1, 3))
        wu = product_rs_velocity(q[0], p[0], t[0], q[2], p[2], t[2], q[1])
        vel, nbr = view_velocities(t, q, p, np.ones(3, np.int32))                  # the NumPy oracle's rule on the same three views
        assert nbr.tolist() == [1, 2, 1] and np.abs(wu - vel[1]).max() < 1e-10
        # one-sided: between the view and its only neighbour
        assert np.abs(product_rs_velocity(q[0], p[0], t[0], q[1], p[1], t[1], q[0]) - vel[0]).max() < 1e-10


# ---- 2. the synthetic sequence: accuracy, velocities, time offset ------------------------------------------------------------------
@pytest.mark.parametrize("model,k", MODELS, ids=MODEL_IDS)
def test_rolling_shutter_poses_are_closer_to_the_truth(model, k):
    """60 fps, 960 x 540, line delay 1/fps/H, ~2.4 rad/s and ~0.6 m/s, 0.2 px noise.  Measured (median over 40 views): position error
    14-16 mm global against 2.1-2.5 mm rolling, rotation error 31-37 mrad against 4.7-5.6 mrad, i.e. a factor 5.5-7.5; asserted: 3."""
    s = rs_sequence(model, k, n_frames=40, seed=model)
    for mode in ("normalized", "tangent"):
        o = _setup(RsPoseOracle(), model, k, s["board"], mode)
        qg, pg, eg, vg = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
        qr, pr, er, vr = _poses(o, s)
        assert vg.all() and vr.all()
        dg, dr = np.median(np.linalg.norm(pg - s["p_wc"], axis=1)), np.median(np.linalg.norm(pr - s["p_wc"], axis=1))
        ag, ar = np.median(_rot_err(qg, s["q_wc"])), np.median(_rot_err(qr, s["q_wc"]))
        assert dr * 3 < dg and ar * 3 < ag, (mode, dg, dr, ag, ar)
        # velocities: central differences over 1/30 s of noisy poses (the two end views are one-sided).  Measured median errors of the inner
        # views: 0.16-0.26 rad/s and 0.07-0.11 m/s, against median speeds of 1.7 rad/s and 0.35 m/s; asserted: 0.4 rad/s and 0.16 m/s
        w, u, n_static = o.pose_velocities(40)
        assert n_static == 0
        inner = slice(1, 39)
        assert np.median(np.linalg.norm(w[inner] - s["w"][inner], axis=1)) < 0.4
        assert np.median(np.linalg.norm(u[inner] - s["u"][inner], axis=1)) < 0.16


def test_time_offset_from_rolling_shutter_poses(oracle_factory):
    """estimate_imu_to_camera_rotation on 480 views (8 s, 0.2 px noise) and a 1 kHz gyroscope whose clock runs 37 ms behind the camera's.
    A global-shutter pose is roughly the pose at the board's mean row time, mean_row * line delay = 8.4 ms after the frame.  The estimator
    cannot show that shift cleanly: its nearest-sample interpolation makes the objective a sawtooth whose minima here lie ~11 ms apart
    (measured on nearby trajectories: -8.53, +2.43, +12.48 ms), the same size as the shift.  Measured on this one: the true poses give
    +2.43 ms, the rolling-shutter poses the same +2.43 ms, the global-shutter poses +406 ms (the search lands in another minimum)."""
    from scipy.spatial.transform import Rotation
    model, k = CASES[0]
    s = rs_sequence(model, k, n_frames=480, seed=3, noise_px=0.2, rot_amp=0.04, pos_amp=0.01, freqs=(0.31, 0.47, 0.71, 0.97, 1.3))
    td0 = 0.037
    R_ic = Rotation.from_rotvec([0.1, -0.2, 0.3]).as_matrix()
    ti = np.arange(s["frame_t"][0] - 0.3, s["frame_t"][-1] + 0.3, 1e-3)
    gyro = np.stack([R_ic @ s["traj"].velocity(t + td0)[0] for t in ti])          # t_cam = t_imu + td
    o = _setup(RsPoseOracle(), model, k, s["board"])
    qg, _, _, vg = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
    qr, _, _, vr = _poses(o, s)
    assert vg.all() and vr.all()
    conj = np.array([-1.0, -1.0, -1.0, 1.0])
    td = {name: oracle_factory().estimate_imu_to_camera_rotation(s["frame_t"], q * conj, ti, gyro, np.zeros(3))["time_offset_s"] - td0
          for name, q in (("truth", s["q_wc"]), ("global", qg), ("rolling", qr))}
    bias = s["mean_row"] * LINE_DELAY
    assert abs(td["truth"]) < 5e-3
    assert abs(td["rolling"] - td["truth"]) < 1e-3 and abs(td["rolling"]) < 5e-3, td
    assert abs(td["global"] - td["truth"]) > 0.5 * bias, (td, bias)


# ---- 3. degenerate cases give back the global-shutter result -----------------------------------------------------------------------
def test_zero_line_delay_and_motionless_camera():
    model, k = CASES[4]
    s = rs_sequence(model, k, n_frames=12, seed=2)
    o = _setup(RsPoseOracle(), model, k, s["board"])
    g = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
    _poses(o, s)
    o.set_pose_rolling_shutter(0.0)
    z = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
    assert all(np.array_equal(a, b) for a, b in zip(g, z))
    # a motionless camera: the rolling-shutter poses are the global-shutter poses
    s = rs_sequence(model, k, n_frames=12, seed=2, noise_px=0.0, rot_amp=0.0, pos_amp=0.0)
    for mode in ("normalized", "tangent"):
        o = _setup(RsPoseOracle(), model, k, s["board"], mode)
        qg, pg, eg, vg = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
        qr, pr, er, vr = _poses(o, s)
        assert (vg == vr).all() and vr.all()
        assert _qdiff(qr, qg).max() < 1e-12 and np.abs(pr - pg).max() < 1e-12


def _gappy(s):
    """the views at 0-3, 4 (alone: 0.25 s from both sides), 5-9 of a 60 fps sequence, in a shuffled order"""
    n = len(s["frame_t"])
    t = s["frame_t"].copy(); t[4] = t[3] + 0.25; t[5:] += 0.5
    perm = np.random.default_rng(0).permutation(n); C = s["board"].shape[0]
    uv = np.concatenate([s["uv"][C * i:C * (i + 1)] for i in perm])
    return dict(s, frame_t=t[perm], uv=uv), perm


def test_views_without_neighbours_keep_the_global_shutter_model():
    model, k = CASES[0]
    s, perm = _gappy(rs_sequence(model, k, n_frames=10, seed=4))
    lone = int(np.nonzero(perm == 4)[0][0])
    o = _setup(RsPoseOracle(), model, k, s["board"])
    qg, pg, eg, vg = o.estimate_board_poses(s["off"], s["ids"], s["uv"])
    qr, pr, er, vr = _poses(o, s)
    w, u, n_static = o.pose_velocities(10)
    assert vr.all() and n_static == 1 and not w[lone].any() and not u[lone].any()
    assert (np.linalg.norm(w, axis=1) > 0).sum() == 9
    assert _qdiff(qr[lone:lone + 1], qg[lone:lone + 1]).max() < 1e-9 and np.abs(pr[lone] - pg[lone]).max() < 1e-9
    others = np.arange(10) != lone
    assert np.abs(pr[others] - pg[others]).min() > 1e-6                           # the rest moved to their frame-time poses


# ---- 4. argument checks ----------------------------------------------------------------------------------------------------------
def test_rolling_shutter_arguments_are_checked_by_the_library():
    from openimucameracalibrator_b200 import calibrator
    h = capi.CApi(calibrator.load_library(), "icc_", -1)                           # host state: a host-only handle takes it
    h.set_pose_rolling_shutter(LINE_DELAY, np.arange(5) / FPS)
    h.set_pose_rolling_shutter(0.0)                                                # global shutter: no times needed
    h.set_pose_rolling_shutter(0.0, np.arange(5) / FPS)
    for ld, t in ((-1e-5, np.arange(5) / FPS), (np.nan, np.arange(5) / FPS), (np.inf, np.arange(5) / FPS), (LINE_DELAY, None),
                  (LINE_DELAY, np.array([0.0, np.nan])), (LINE_DELAY, np.array([0.0, -0.1])), (LINE_DELAY, np.zeros(0))):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
            h.set_pose_rolling_shutter(ld, t)
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.pose_velocities(5)
    # the next pose call must pass the same number of views
    model, k = CASES[0]
    s = rs_sequence(model, k, n_frames=4, seed=1)
    _setup(h, model, k, s["board"])
    h.set_pose_rolling_shutter(LINE_DELAY, np.arange(5) / FPS)
    for call in (lambda: h.estimate_board_poses(s["off"], s["ids"], s["uv"]),
                 lambda: h.optimize_board_points(s["off"], s["ids"], s["uv"], s["q_wc"], s["p_wc"], np.ones(4, np.int32))):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT.*n_frames"):
            call()
    h.set_pose_rolling_shutter(LINE_DELAY, s["frame_t"])
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h.estimate_board_poses(s["off"], s["ids"], s["uv"])
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):                      # a failed call leaves no velocities behind
        h.pose_velocities(4)
    o = _setup(RsPoseOracle(), model, k, s["board"])
    o.set_pose_rolling_shutter(LINE_DELAY, np.arange(5) / FPS)
    with pytest.raises(ValueError):
        o.estimate_board_poses(s["off"], s["ids"], s["uv"])


def test_pose_shutter_flag_is_parsed_and_checked(tmp_path):
    for cli in (POSE_CLI, HOT_CLI):
        assert os.path.exists(cli), "build the CLI first (__graft_entry__.build())"
        for bad in ("--pose_shutter=Rolling", "--pose_shutter=rs", "--pose_shutter="):
            out = subprocess.run([cli, bad], capture_output=True, text=True)
            assert out.returncode == 1 and "--pose_shutter must be 'global' or 'rolling'" in out.stderr, (cli, bad, out.stderr)
    ds = syn.make_dataset(syn.tiny_config())
    paths = iof.write_dataset_files(ds, str(tmp_path))
    base = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items() if a != "input_pose_dataset"] + ["--parse_only"]
    runs = [subprocess.run(base + extra, capture_output=True, text=True) for extra in ([], ["--pose_shutter=global"], ["--pose_shutter", "rolling"])]
    assert all(r.returncode == 0 for r in runs), [r.stderr for r in runs]
    assert runs[0].stdout == runs[1].stdout == runs[2].stdout
    for extra in (["--global_shutter"], ["--input_pose_dataset=" + paths["input_pose_dataset"]]):
        out = subprocess.run(base + ["--pose_shutter=rolling"] + extra, capture_output=True, text=True)
        assert out.returncode == 1 and "--pose_shutter rolling" in out.stderr, (extra, out.stderr)
    # fps <= 0 in the camera calibration is a usage error of --pose_shutter rolling
    cam = json.load(open(paths["camera_calibration_json"]))
    assert "fps" in cam
    cam["fps"] = 0.0
    bad_cam = str(tmp_path / "cam_fps0.json"); json.dump(cam, open(bad_cam, "w"))
    out = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + bad_cam, "--pose_shutter=rolling"],
                         capture_output=True, text=True)
    assert out.returncode == 1 and "fps > 0" in out.stderr, out.stderr


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------
# Both sides stop when the cost stalls at 1e-15 relative, which pins the pose of a noisy view to ~1e-9 (measured up to 3.6e-9 here): the
# project's bound for GPU against oracle on noisy views is 2e-8 (test_pose_estimation.py).  Velocities are differences of poses 1/30 s
# apart, so 2e-8 in the poses is up to ~1.2e-6 in them.
TOL, VTOL = 2e-8, 2e-6


def _gpu_and_oracle(g, o, s):
    """The GPU's rolling-shutter poses and the oracle's two rolling-shutter passes started from the GPU's own global-shutter pass.
    The global-shutter pass is the unchanged default path (a zero line delay runs it alone, bit for bit as inside the rolling call); on
    these skewed views its GPU and oracle optima can sit up to ~1e-4 apart on some views of some cameras (measured on FOV and
    PinholeRadialTangential, every model within 2e-8 on global-shutter scenes), and the rolling passes carry that difference along.
    Starting both from the same poses holds the new passes themselves to TOL."""
    g.set_pose_rolling_shutter(0.0)
    gs = g.estimate_board_poses(s["off"], s["ids"], s["uv"])
    rg = _poses(g, s)
    o.set_pose_rolling_shutter(LINE_DELAY, s["frame_t"])
    ro = o.rolling_passes(s["off"], s["ids"], s["uv"], gs)
    return rg, ro


def _compare(a, b, tol):
    """(q, p, e, v) of two implementations: validity bit for bit, poses and mean errors to tol"""
    assert (a[3] == b[3]).all()
    d = max(_qdiff(a[0], b[0]).max(), np.abs(a[1] - b[1]).max(), np.abs(a[2] - b[2]).max())
    print(f"\n[rolling shutter parity] max difference {d:.3g}")
    assert d < tol


@pytest.mark.gpu
@pytest.mark.parametrize("model,k", CASES, ids=ALL_IDS)
def test_gpu_rolling_shutter_poses_match_oracle(gpu_factory, model, k):
    s = rs_sequence(model, k, n_frames=30, seed=model + 90)
    s["uv"][s["off"][7] + 11] += 60.0                                              # one gross outlier in view 7
    for mode in ("normalized", "tangent"):
        o, g = _setup(RsPoseOracle(), model, k, s["board"], mode), _setup(gpu_factory(), model, k, s["board"], mode)
        rg, ro = _gpu_and_oracle(g, o, s)
        assert ro[3].all()
        _compare(rg, ro, TOL)
        wo, uo, no = o.pose_velocities(30); wg, ug, ng = g.pose_velocities(30)
        assert ng == no == 0 and np.abs(wg - wo).max() < VTOL and np.abs(ug - uo).max() < VTOL


@pytest.mark.gpu
def test_gpu_zero_delay_and_lone_views(gpu_factory):
    model, k = CASES[0]
    s, perm = _gappy(rs_sequence(model, k, n_frames=10, seed=4))
    g = _setup(gpu_factory(), model, k, s["board"])
    ref = g.estimate_board_poses(s["off"], s["ids"], s["uv"])
    rg = _poses(g, s)
    g.set_pose_rolling_shutter(0.0)
    z = g.estimate_board_poses(s["off"], s["ids"], s["uv"])
    assert all(np.array_equal(a, b) for a, b in zip(ref, z))                         # a zero line delay: today's outputs bit for bit
    o = _setup(RsPoseOracle(), model, k, s["board"])
    o.set_pose_rolling_shutter(LINE_DELAY, s["frame_t"])
    ro = o.rolling_passes(s["off"], s["ids"], s["uv"], ref)
    _compare(rg, ro, TOL)
    wg, ug, ng = g.pose_velocities(10); wo, uo, no = o.pose_velocities(10)
    lone = int(np.nonzero(perm == 4)[0][0])
    assert ng == no == 1 and not wg[lone].any() and not ug[lone].any() and np.abs(wg - wo).max() < VTOL and np.abs(ug - uo).max() < VTOL


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["normalized", "tangent"])
def test_gpu_rolling_shutter_board_points_match_oracle(gpu_factory, mode):
    model, k = CASES[4]
    s = rs_sequence(model, k, n_frames=50, seed=6, noise_px=0.1)
    bad = s["board"].copy(); bad[:, :3] += np.random.default_rng(1).normal(0, 5e-4, (bad.shape[0], 3))
    o, g = _setup(RsPoseOracle(), model, k, bad, mode), _setup(gpu_factory(), model, k, bad, mode)
    (qg, pg, eg, vg), ro = _gpu_and_oracle(g, o, s)
    _compare((qg, pg, eg, vg), ro, TOL)
    # both from the GPU's rolling-shutter poses
    ro = o.optimize_board_points(s["off"], s["ids"], s["uv"], qg, pg, vg, min_observations=20)
    rg = g.optimize_board_points(s["off"], s["ids"], s["uv"], qg, pg, vg, min_observations=20)
    assert rg[5] == ro[5] == bad.shape[0]
    _compare(rg[:4], ro[:4], TOL)
    assert np.abs(rg[4] - ro[4]).max() < TOL and rg[2].mean() < eg.mean()
    wo, uo, _ = o.pose_velocities(50); wg, ug, _ = g.pose_velocities(50)
    assert np.abs(wg - wo).max() < VTOL and np.abs(ug - uo).max() < VTOL


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                                               # noqa: BLE001 - the reading is informative only
        pl = "unknown"
    return f"{name}, power limit {pl or 'unknown'}"


@pytest.mark.gpu
def test_gpu_rolling_shutter_full_size(gpu_factory):
    """3000 views x 144 corners: every view valid, a 30-view sample equals the oracle; wall time of the pose step, global against rolling."""
    import time
    from rolling_shutter_support import board as make_board
    model, k = CASES[4]
    B = make_board(12, 12, 0.015)
    # 3000 views: the 30-view sequence's poses at 100 times its length (views 1/60 s apart), corners of the 12 x 12 board from the true poses
    # at each corner's row time is too slow to generate here, so the large scene uses the global-shutter projection of a smooth trajectory
    from rolling_shutter_support import Trajectory
    traj = Trajectory(7, rot_amp=0.08, pos_amp=0.02, freqs=(0.3, 0.5, 0.7, 0.9, 1.1))
    n = 3000; C = B.shape[0]
    t = 1.0 + np.arange(n) / FPS
    uv = []
    rng = np.random.default_rng(0)
    for tf in t:
        pc = (B[:, :3] - traj.p(tf)) @ traj.R(tf)
        px, valid = cm.project(model, k, pc)
        assert valid.all()
        uv.append(px + rng.normal(0, 0.2, px.shape))
    uv = np.concatenate(uv); off = (np.arange(n + 1) * C).astype(np.int32); ids = np.tile(np.arange(C, dtype=np.int32), n)
    g = _setup(gpu_factory(), model, k, B)
    g.estimate_board_poses(off, ids, uv)                                           # warm-up
    t0 = time.perf_counter(); rgl = g.estimate_board_poses(off, ids, uv); dt_g = time.perf_counter() - t0
    g.set_pose_rolling_shutter(LINE_DELAY, t)
    g.estimate_board_poses(off, ids, uv)
    t0 = time.perf_counter(); rr = g.estimate_board_poses(off, ids, uv); dt_r = time.perf_counter() - t0
    assert rgl[3].all() and rr[3].all()
    o = _setup(RsPoseOracle(), model, k, B)
    m = 30
    o.set_pose_rolling_shutter(LINE_DELAY, t[:m])
    ro = o.rolling_passes(off[: m + 1], ids[: off[m]], uv[: off[m]], [x[:m] for x in rgl])      # from the GPU's global-shutter poses
    # the sample's last view has one neighbour in the sample but two in the full run, which reaches its neighbours' velocities in the
    # second pass: compare the views whose neighbours' poses agree in both passes
    assert ro[3].all() and _qdiff(rr[0][:m - 3], ro[0][:m - 3]).max() < TOL and np.abs(rr[1][:m - 3] - ro[1][:m - 3]).max() < TOL
    line = f"[f1 rolling shutter] 3000 views x 144 corners, {_card()}: pose step {dt_g * 1e3:.2f} ms global, {dt_r * 1e3:.2f} ms rolling (wall, incl. H2D/D2H)"
    print("\n" + line)


@pytest.mark.gpu
def test_gpu_tool_chain_with_rolling_shutter(tmp_path, gpu_factory):
    """pose CLI --pose_shutter rolling -> rotation CLI -> hot CLI, through the files the tools exchange."""
    from test_cli_formats import _args
    cfg = syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), n_frames=600, grid=(8, 6), imu_rate_hz=400.0, seed=5)
    ds = syn.make_dataset(cfg)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    outs = {}
    for shutter in ("global", "rolling"):
        pose_json, init_json = str(tmp_path / f"poses_{shutter}.json"), str(tmp_path / f"init_{shutter}.json")
        r = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + paths["camera_calibration_json"],
                            "--output_pose_dataset=" + pose_json, "--pose_shutter=" + shutter], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr + r.stdout
        assert ("Rolling shutter: line delay" in r.stdout) == (shutter == "rolling")
        r = subprocess.run([ROT_CLI, "--input_pose_calibration_dataset=" + pose_json, "--telemetry_json=" + paths["telemetry_json"],
                            "--imu_rotation_init_output=" + init_json], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr + r.stdout
        outs[shutter] = (json.load(open(pose_json)), json.load(open(init_json)))
    pg, pr = outs["global"][0], outs["rolling"][0]
    assert set(pr["views"]) <= set(pg["views"]) and len(pr["views"]) >= 0.95 * len(pg["views"])
    assert set(next(iter(pr["views"].values()))) == set(next(iter(pg["views"].values())))      # the pose dataset keeps its format
    print(f"\n[rolling shutter tool chain] time offset: global {outs['global'][1]['time_offset_gyro_to_cam']:.5f} s, "
          f"rolling {outs['rolling'][1]['time_offset_gyro_to_cam']:.5f} s, truth {ds['time_offset_imu_to_cam_s']:.5f} s")
    assert abs(outs["rolling"][1]["time_offset_gyro_to_cam"] - ds["time_offset_imu_to_cam_s"]) < 0.03
    pth = dict(paths, input_pose_dataset=str(tmp_path / "poses_rolling.json"), gyro_to_cam_initial_calibration=str(tmp_path / "init_rolling.json"))
    r = subprocess.run(_args(pth, str(tmp_path)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    res = iof.read_result_json(str(tmp_path / "result.json"))
    assert np.isfinite(res["final_reproj_error"])
    # the in-process pose step of the hot CLI takes the flag as well
    args = [a for a in _args(dict(paths, gyro_to_cam_initial_calibration=str(tmp_path / "init_rolling.json")), str(tmp_path)) if not a.startswith("--input_pose_dataset")]
    r = subprocess.run(args + ["--pose_shutter=rolling"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "Estimated board poses for" in r.stdout
