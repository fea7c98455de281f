"""Rolling-shutter camera calibration (icc_set_camcal_rolling_shutter): intrinsics and view poses from row-timed corners.

Corner c of view i is seen tau = uv_c.y * line_delay after its frame and predicted from P(tau) = exp(-tau [w_i]x) (R_cw (X - c_wc) - tau u_i),
the model of the pose step's rolling shutter, with the view's velocities held fixed in each bundle adjustment.

- Rows: the product's rs_camera_residual compiled for the CPU (tests/rolling_shutter/rs_camcal_host_math.cu) against central differences, and
  against the global-shutter rows with w = u = 0.
- Oracle: tests/rolling_shutter/rs_camcal_oracle.cpp, the unchanged C++ oracle with its bundle-adjustment residual and its board-point
  observation swapped for rolling-shutter versions (fixed mode).  The automatic mode's oracle is composed here: the oracle's global-shutter
  calibration, then `RsPoseOracle` poses and velocities under those intrinsics, then the rolling-shutter oracle, twice.
- Data: a sequence with a physical rolling shutter (rolling_shutter_support: every corner projected with the true pose at its own row time).
"""
import ctypes
import json
import os
import subprocess
import tempfile
import time

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_calibration import CASES, IDS, TIGHT, _bent, _qdiff, scene
from test_camera_models import CASES as MODEL_CASES
from rolling_shutter_support import FPS, LINE_DELAY, RsPoseOracle, rs_sequence

HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(os.path.dirname(HERE), "openimucameracalibrator_b200", "bin")
CAL_CLI = os.path.join(BIN, "calibrate_camera")
POSE_CLI = os.path.join(BIN, "estimate_camera_poses_from_checkerboard")
ROT_CLI = os.path.join(BIN, "estimate_imu_to_camera_rotation")
W, H = 960, 540
GPU_CASES = CASES + [(cm.PINHOLE_RADIAL_TANGENTIAL, MODEL_CASES[-1][1])]
GPU_IDS = IDS + ["PINHOLE_RADIAL_TANGENTIAL"]
_LIBS = {}


def _build(name, cmd_of):
    if name not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_rs_camcal_"), f"lib{name}.so")
        subprocess.check_call(cmd_of(out))
        _LIBS[name] = ctypes.CDLL(out)
    return _LIBS[name]


def host_math_lib():
    return _build("rs_camcal_host_math", lambda out: ["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                                                      "-o", out, os.path.join(HERE, "rolling_shutter", "rs_camcal_host_math.cu")])


def rs_oracle():
    """the CPU oracle with the rolling-shutter residuals (fixed mode), built once per process"""
    lib = _build("rs_camcal_oracle", lambda out: ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out,
                                                  os.path.join(HERE, "rolling_shutter", "rs_camcal_oracle.cpp")])
    return capi.CApi(lib, "icco_", 0)


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _c(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def product_rows(model, k, q, c, X, wu, tau, uv):
    """-> (r[2], ok, J[2,6], Jk[2,10]) of rs_camera_residual; q = R_cw (x,y,z,w)"""
    kk = np.zeros(10); kk[:len(k)] = k
    r = np.zeros(2); J = np.zeros(12); Jk = np.zeros(20)
    lib = host_math_lib(); lib.rs_camera_rows.restype = ctypes.c_int
    ok = lib.rs_camera_rows(int(model), *[_dp(_c(v)) for v in (kk, q, c, X, wu)], ctypes.c_double(tau), _dp(_c(uv)), _dp(r), _dp(J), _dp(Jk))
    return r, bool(ok), J.reshape(2, 6), Jk.reshape(2, 10)


def gs_rows(model, k, q, c, X, uv):
    kk = np.zeros(10); kk[:len(k)] = k
    r = np.zeros(2); J = np.zeros(12); Jk = np.zeros(20)
    lib = host_math_lib(); lib.gs_camera_rows.restype = ctypes.c_int
    ok = lib.gs_camera_rows(int(model), *[_dp(_c(v)) for v in (kk, q, c, X, uv)], _dp(r), _dp(J), _dp(Jk))
    return r, bool(ok), J.reshape(2, 6), Jk.reshape(2, 10)


def rs_project(model, k, q_wc, p_wc, wu, X, line_delay):
    """pixels of board points X under the constant-velocity rolling-shutter model (fixed point in the row)"""
    P0 = (X - p_wc) @ Rotation.from_quat(q_wc).as_matrix()
    tau = np.zeros(len(X))
    for _ in range(10):
        A = Rotation.from_rotvec(-tau[:, None] * wu[None, :3]).as_matrix()
        px, valid = cm.project(model, k, np.einsum("nij,nj->ni", A, P0 - tau[:, None] * wu[None, 3:]))
        tau = px[:, 1] * line_delay
    return px, valid


def rs_scene(model, k, n_views=36, seed=0, noise_px=0.2, grid=(9, 7)):
    """the views of test_camera_calibration.scene, seen through the constant-velocity rolling-shutter model with random velocities
    (|w| about 1.7 rad/s, |u| about 0.26 m/s) -> (board, off, ids, uv, vel[n,6])"""
    B, off, ids, _, q, p = scene(model, k, n_views=n_views, seed=seed, grid=grid)
    rng = np.random.default_rng(seed + 500)
    vel = np.concatenate([rng.normal(0, 1.0, (n_views, 3)), rng.normal(0, 0.15, (n_views, 3))], 1)
    uv = np.concatenate([rs_project(model, k, q[i], p[i], vel[i], B[:, :3], LINE_DELAY)[0] for i in range(n_views)])
    return B, off, ids, uv + rng.normal(0, noise_px, uv.shape), vel


# The physical sequence of the truth tests: 60 views at 60 fps, rotations up to 0.45 rad about the looking-down pose at 0.7-1.1 Hz, so up to
# 2.8 rad/s; 0.1 px noise.
PHYS = dict(n_frames=60, seed=3, noise_px=0.1, rot_amp=0.45, pos_amp=0.03, freqs=(0.7, 1.1))
TRUTH_MODELS = [(m, k) for m, k in CASES if m in (cm.PINHOLE, cm.EXTENDED_UNIFIED)]


def _groups(model, d):
    """|intrinsic error| per group: focal length, principal point, distortion (Theia order)"""
    d = np.abs(np.asarray(d))
    noskew = model in (cm.FOV, cm.DIVISION_UNDISTORTION)
    pp = d[2:4] if noskew else d[3:5]
    dist = d[4:5] if noskew else d[5:cm.NUM_PARAMS[model]]
    return np.array([d[0], pp.max(), dist.max()])


def _calibrate(api, model, s, **kw):
    api.set_board_points(s["board"])
    return api.calibrate_camera(model, W, H, s["off"], s["ids"], s["uv"], grid_size=0.0, **TIGHT, **kw)


def composed_oracle(model, s, board, frame_t, **kw):
    """the automatic mode on the CPU: the oracle's global-shutter calibration, then twice the rolling-shutter pose oracle under the last
    intrinsics and the rolling-shutter oracle with its velocities (zero for views it could not place) -> (result, vel, n_static)"""
    o = rs_oracle(); o.set_board_points(board)
    r = o.calibrate_camera(model, W, H, s["off"], s["ids"], s["uv"], **kw)
    if not r["summary"]["success"]:
        return r, None, 0
    for _ in range(2):
        po = RsPoseOracle(); po.set_camera(model, r["intrinsics"], W, H); po.set_board_points(board); po.set_pose_rolling_shutter(LINE_DELAY, frame_t)
        _, _, _, v = po.estimate_board_poses(s["off"], s["ids"], s["uv"], 0.0, 0)
        vel = po.vel.copy(); vel[v == 0] = 0.0
        o = rs_oracle(); o.set_board_points(board); o.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
        r = o.calibrate_camera(model, W, H, s["off"], s["ids"], s["uv"], **kw)
    return r, vel, po.n_static


# ---- 1. rows -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,k", MODEL_CASES, ids=[cm.MODEL_NAMES[m] for m, _ in MODEL_CASES])
def test_rs_camera_rows_against_central_differences(model, k):
    rng = np.random.default_rng(model + 3)
    n = cm.NUM_PARAMS[model]
    for _ in range(5):
        R_wc = Rotation.from_rotvec(np.array([np.pi, 0, 0]) + rng.normal(0, 0.3, 3)).as_matrix()
        c = np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(0.3, 0.45)])
        X = np.array([rng.uniform(-0.08, 0.08), rng.uniform(-0.06, 0.06), 0.0])
        q = Rotation.from_matrix(R_wc.T).as_quat()                                          # R_cw
        wu = np.r_[rng.normal(0, 2.0, 3), rng.normal(0, 0.3, 3)]
        uv = np.array([400.0, 300.0]); tau = 300.0 * LINE_DELAY
        r, ok, J, Jk = product_rows(model, k, q, c, X, wu, tau, uv)
        assert ok
        hs = 1e-6
        for j in range(6):                                                                  # right increment on R_cw, then the camera centre
            def at(sg):
                if j < 3:
                    e = np.zeros(3); e[j] = sg * hs
                    return product_rows(model, k, Rotation.from_matrix(R_wc.T @ Rotation.from_rotvec(e).as_matrix()).as_quat(), c, X, wu, tau, uv)[0]
                cc = c.copy(); cc[j - 3] += sg * hs
                return product_rows(model, k, q, cc, X, wu, tau, uv)[0]
            assert np.abs((at(1) - at(-1)) / (2 * hs) - J[:, j]).max() < 1e-5 * max(1.0, np.abs(J).max())
        for i in range(n):
            h = 1e-6 * abs(k[i]) if k[i] != 0 else 1e-7                                  # relative steps: the division model's k is ~1e-7
            kp, km = np.array(k, dtype=np.float64), np.array(k, dtype=np.float64); kp[i] += h; km[i] -= h
            d = (product_rows(model, kp, q, c, X, wu, tau, uv)[0] - product_rows(model, km, q, c, X, wu, tau, uv)[0]) / (2 * h)
            assert np.abs(d - Jk[:, i]).max() < 1e-5 * max(1.0, np.abs(Jk[:, i]).max()), (i, d, Jk[:, i])
        assert not Jk[:, n:].any()
        # without motion: the global-shutter rows, whatever the row time
        r0, ok0, J0, Jk0 = product_rows(model, k, q, c, X, np.zeros(6), tau, uv)
        rg, okg, Jg, Jkg = gs_rows(model, k, q, c, X, uv)
        assert ok0 == okg and np.array_equal(r0, rg) and np.array_equal(J0, Jg) and np.array_equal(Jk0, Jkg)


# ---- 2. the oracle on a physical rolling shutter --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,k", TRUTH_MODELS, ids=[cm.MODEL_NAMES[m] for m, _ in TRUTH_MODELS])
def test_oracle_rolling_shutter_recovers_the_truth_the_global_shutter_misses(model, k):
    """Measured with this file's oracle (PHYS, true velocities), |error| of focal length / principal point / distortion:
         PINHOLE           global 100.8 px / 31.7 px / 5.2e-2    rolling 0.59 px / 1.41 px / 1.2e-3
         EXTENDED_UNIFIED  global 207.8 px / 107 px / 0.44       rolling 0.72 px / 1.62 px / 5.8e-2
       The premise (global focal length off by more than 50 px) and a factor of 4 in every group are asserted."""
    s = rs_sequence(model, k, **PHYS)
    vel = np.concatenate([s["w"], s["u"]], 1)
    gs = _calibrate(rs_oracle(), model, s)
    o = rs_oracle(); o.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    rs = _calibrate(o, model, s)
    eg, er = _groups(model, gs["intrinsics"] - k), _groups(model, rs["intrinsics"] - k)
    print(f"\n[rs camcal truth] {cm.MODEL_NAMES[model]}: global {eg}, rolling {er}; mean errors {gs['summary']['final_reproj_error']:.3f} / "
          f"{rs['summary']['final_reproj_error']:.3f} px")
    assert eg[0] > 50.0                                                                      # the premise: the global shutter is biased
    assert (er * 4 < eg).all()
    assert rs["summary"]["success"] == 1 and (rs["used"] >= gs["used"]).all()
    assert rs["summary"]["final_reproj_error"] < 0.15                                        # 0.1 px noise per axis: mean norm ~0.125 px


def test_oracle_with_zero_velocities_is_the_global_shutter():
    model, k = CASES[4]
    B, off, ids, uv, vel = rs_scene(model, k, n_views=24, seed=9)
    s = dict(board=B, off=off, ids=ids, uv=uv)
    gs = _calibrate(rs_oracle(), model, s)
    o = rs_oracle(); o.set_camcal_rolling_shutter(LINE_DELAY, w_u=np.zeros_like(vel))
    z = _calibrate(o, model, s)
    assert (z["used"] == gs["used"]).all()
    assert np.abs(z["intrinsics"] - gs["intrinsics"]).max() <= 1e-12 * np.abs(gs["intrinsics"]).max()
    assert _qdiff(z["q_wc"], gs["q_wc"]).max() <= 1e-12 and np.abs(z["p_wc"] - gs["p_wc"]).max() <= 1e-12
    # and the fixed velocities of the data do move it
    o.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    r = _calibrate(o, model, s)
    assert r["summary"]["final_reproj_error"] < gs["summary"]["final_reproj_error"]


# ---- 3. arguments and the command line ----------------------------------------------------------------------------------------------------------
def test_camcal_rolling_shutter_arguments_are_checked_by_the_library():
    from openimucameracalibrator_b200 import calibrator
    h = capi.CApi(calibrator.load_library(), "icc_", -1)                                   # host state: a host-only handle takes it
    t = np.arange(5) / FPS
    h.set_camcal_rolling_shutter(LINE_DELAY, frame_t_s=t)
    h.set_camcal_rolling_shutter(LINE_DELAY, w_u=np.zeros((5, 6)))
    h.set_camcal_rolling_shutter(0.0)
    for ld, tt, wu in ((-1e-5, t, None), (np.nan, t, None), (np.inf, None, np.zeros((5, 6))), (LINE_DELAY, None, None),
                       (LINE_DELAY, np.array([0.0, np.nan]), None), (LINE_DELAY, np.array([0.0, -0.1]), None), (LINE_DELAY, np.zeros(0), None),
                       (LINE_DELAY, None, np.array([[0, 0, np.inf, 0, 0, 0]]))):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
            h.set_camcal_rolling_shutter(ld, frame_t_s=tt, w_u=wu)
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.camcal_velocities(5)
    model, k = CASES[0]
    B, off, ids, uv, q, p = scene(model, k, n_views=4, seed=1)
    h.set_board_points(B)
    h.set_camcal_rolling_shutter(LINE_DELAY, frame_t_s=t)                                  # 5 views, the call passes 4
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT.*n_views"):
        h.calibrate_camera(model, W, H, off, ids, uv)
    h.set_camcal_rolling_shutter(LINE_DELAY, frame_t_s=t[:4])
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h.calibrate_camera(model, W, H, off, ids, uv)
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.camcal_velocities(4)
    # the pose step's shutter is separate state
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.pose_velocities(4)


def _corner_file(path, s, fps=FPS, height=H):
    scene_json = {"camera_fps": float(fps), "image_width": W, "image_height": height,
                  "scene_pts": {str(i): list(map(float, b[:3])) for i, b in enumerate(s["board"])},
                  "views": {f"{t * 1e6:.6f}": {"image_points": {str(int(s["ids"][c])): [float(s["uv"][c, 0]), float(s["uv"][c, 1])]
                                                                for c in range(s["off"][f], s["off"][f + 1])}} for f, t in enumerate(s["frame_t"])}}
    with open(path, "wb") as f:
        f.write(iof.ubjson_dumps(scene_json))
    return scene_json


def test_calibrate_camera_pose_shutter_flag_is_parsed_and_checked(tmp_path):
    assert os.path.exists(CAL_CLI), "build the CLI first (__graft_entry__.build())"
    for bad in ("--pose_shutter=Rolling", "--pose_shutter=rs", "--pose_shutter="):
        out = subprocess.run([CAL_CLI, bad], capture_output=True, text=True)
        assert out.returncode == 1 and "--pose_shutter must be 'global' or 'rolling'" in out.stderr, (bad, out.stderr)
    model, k = CASES[0]
    s = rs_sequence(model, k, n_frames=4, seed=1)
    _corner_file(str(tmp_path / "fps0.uson"), s, fps=0.0)
    out = subprocess.run([CAL_CLI, "--input_corners=" + str(tmp_path / "fps0.uson"), "--camera_model_to_calibrate=PINHOLE", "--pose_shutter=rolling"],
                         capture_output=True, text=True)
    assert out.returncode == 1 and "fps > 0" in out.stderr, out.stderr


# ---- 4. GPU -------------------------------------------------------------------------------------------------------------------------------------
def _parity(rg, ro, model, pose_tol=1e-7, view_tol=1e-6, cost_tol=1e-7):
    so, sg = ro["summary"], rg["summary"]
    assert sg["success"] == so["success"] == 1 and (rg["used"] == ro["used"]).all()
    n = cm.NUM_PARAMS[model]
    scale = np.maximum(np.abs(ro["intrinsics"]), 1e-3 * np.abs(ro["intrinsics"]).max())
    d = (np.abs(rg["intrinsics"] - ro["intrinsics"])[:n] / scale[:n]).max()
    print(f"\n[rs camcal parity] {cm.MODEL_NAMES[model]}: intrinsics {d:.3g}, poses {_qdiff(rg['q_wc'], ro['q_wc']).max():.3g} / "
          f"{np.abs(rg['p_wc'] - ro['p_wc']).max():.3g}")
    assert d < 1e-6
    assert _qdiff(rg["q_wc"], ro["q_wc"]).max() < pose_tol and np.abs(rg["p_wc"] - ro["p_wc"]).max() < pose_tol
    assert np.abs(rg["view_error_px"] - ro["view_error_px"]).max() < view_tol
    assert abs(sg["final_cost"][2] - so["final_cost"][2]) < cost_tol * so["final_cost"][2]


@pytest.mark.gpu
@pytest.mark.parametrize("obp", [0, 1], ids=["views", "board_points"])
@pytest.mark.parametrize("model,k", GPU_CASES, ids=GPU_IDS)
def test_gpu_fixed_mode_matches_oracle(oracle_factory, gpu_factory, model, k, obp):
    B, off, ids, uv, vel = rs_scene(model, k, n_views=36, seed=model + 60)
    uv[off[5] + 7] += 25.0                                                                   # a gross outlier inside the Huber tail
    board = _bent(B) if obp else B
    s = dict(board=board, off=off, ids=ids, uv=uv)
    o, g = rs_oracle(), gpu_factory()
    for a in (o, g):
        a.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    ro, rg = _calibrate(o, model, s, optimize_board_points=obp), _calibrate(g, model, s, optimize_board_points=obp)
    _parity(rg, ro, model)
    if obp:
        assert rg["summary"]["n_points_optimized"] == ro["summary"]["n_points_optimized"] == B.shape[0]
        assert np.abs(g.get_board_points() - o.get_board_points()).max() < 1e-7
    wg, ug, ng = g.camcal_velocities(36)
    assert np.array_equal(np.concatenate([wg, ug], 1), vel) and ng == 0


@pytest.mark.gpu
def test_gpu_automatic_mode_matches_composed_oracle(gpu_factory):
    model, k = CASES[4]
    s = rs_sequence(model, k, **PHYS)
    s["uv"][s["off"][9] + 4] += 25.0
    ro, vo, no = composed_oracle(model, s, s["board"], s["frame_t"], grid_size=0.0, **TIGHT)
    g = gpu_factory(); g.set_camcal_rolling_shutter(LINE_DELAY, frame_t_s=s["frame_t"])
    rg = _calibrate(g, model, s)
    # the velocities come from the GPU pose step and from the NumPy pose oracle, which agree to about 1e-6 (test_rolling_shutter_poses' VTOL);
    # measured on an H100: intrinsics 7.4e-8 relative, poses 1.8e-7 / 1.9e-7, view errors 2.5e-6 px; held to ten times the fixed mode's bars
    _parity(rg, ro, model, pose_tol=1e-6, view_tol=1e-5, cost_tol=1e-6)
    wg, ug, ng = g.camcal_velocities(len(s["frame_t"]))
    dv = np.abs(np.concatenate([wg, ug], 1) - vo).max()
    print(f"[rs camcal automatic] velocities {dv:.3g}")
    assert ng == no and dv < 2e-4                                                            # measured 3.9e-5 against up to 2.8 rad/s
    # the truth: two rounds from the biased global-shutter start do not reach what the true velocities give (0.7 px of focal length), but every
    # group moves well towards it.  Measured on an H100 (focal length / principal point / distortion): global 207.6 px / 107.3 px / 0.46,
    # automatic 29.3 px / 23.9 px / 0.13, i.e. 7.1x / 4.5x / 3.5x closer; 2x is asserted
    gs = _calibrate(gpu_factory(), model, s)
    eg, er = _groups(model, gs["intrinsics"] - k), _groups(model, rg["intrinsics"] - k)
    print(f"[rs camcal automatic truth] global {eg}, rolling {er}")
    assert (er * 2 < eg).all()


@pytest.mark.gpu
def test_gpu_zero_velocities_and_zero_delay(gpu_factory):
    model, k = CASES[1]
    B, off, ids, uv, vel = rs_scene(model, k, n_views=30, seed=17)
    # The normal equations are summed with RED.ADD, so two runs differ in their last bits, and with tolerances a run may stop one iteration
    # earlier or later (3e-7 px of focal length apart, measured).  These comparisons therefore run a fixed number of iterations per stage.
    opts = dict(function_tolerance=1e-300, parameter_tolerance=1e-300, gradient_tolerance=1e-300, max_num_iterations=12)
    run = lambda api: api.calibrate_camera(model, W, H, off, ids, uv, grid_size=0.0, **opts)   # noqa: E731
    ref = []
    for _ in range(2):
        a = gpu_factory(); a.set_board_points(B); ref.append(run(a))
    g = gpu_factory(); g.set_board_points(B); g.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel); g.set_camcal_rolling_shutter(0.0)
    z = run(g)
    # a zero delay runs today's kernels: its outputs differ from a default run no more than two default runs do
    for key in ("intrinsics", "q_wc", "p_wc", "view_error_px"):
        scatter = np.abs(ref[0][key] - ref[1][key]).max()
        d = np.abs(z[key] - ref[0][key]).max()
        print(f"\n[rs camcal zero delay] {key}: {d:.3g} (two default runs: {scatter:.3g})")
        assert d <= max(scatter, 1e-12 * np.abs(ref[0][key]).max()), (key, d, scatter)
    assert (z["used"] == ref[0]["used"]).all()
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        g.camcal_velocities(30)
    g.set_camcal_rolling_shutter(LINE_DELAY, w_u=np.zeros((30, 6)))
    r0 = run(g)
    d = np.abs(r0["intrinsics"] - ref[0]["intrinsics"]).max() / np.abs(ref[0]["intrinsics"]).max()
    print(f"\n[rs camcal zero velocities] intrinsics {d:.3g} relative")
    assert (r0["used"] == ref[0]["used"]).all() and d < 1e-12
    assert _qdiff(r0["q_wc"], ref[0]["q_wc"]).max() < 1e-12 and np.abs(r0["p_wc"] - ref[0]["p_wc"]).max() < 1e-12


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                                                         # noqa: BLE001 - the reading is informative only
        pl = "unknown"
    return f"{name}, power limit {pl or 'unknown'}"


@pytest.mark.gpu
def test_gpu_rolling_shutter_full_size(gpu_factory):
    """3000 views x 144 corners (the size of test_gpu_calibration_full_size), fixed mode: wall time of the global and the rolling-shutter
    calibration, reported, not asserted."""
    model, k = CASES[4]
    B, off, ids, uv, vel = rs_scene(model, k, n_views=3000, seed=123, grid=(16, 9))
    s = dict(board=B, off=off, ids=ids, uv=uv)
    g = gpu_factory(); g.set_board_points(B)
    small = dict(board=B, off=off[:41], ids=ids[: off[40]], uv=uv[: off[40]])
    _calibrate(g, model, small)                                                              # warm-up (allocations, module load)
    t0 = time.perf_counter(); rgs = g.calibrate_camera(model, W, H, off, ids, uv, grid_size=0.0); dt_g = time.perf_counter() - t0
    g.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel[:40]); _calibrate(g, model, small)
    g.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    t0 = time.perf_counter(); rrs = g.calibrate_camera(model, W, H, off, ids, uv, grid_size=0.0); dt_r = time.perf_counter() - t0
    assert rrs["summary"]["success"] == 1 and rrs["summary"]["n_views_used"] == 3000
    assert np.abs(rrs["intrinsics"] - k).max() < 2e-3 * np.abs(k).max()
    assert 0.2 < rrs["summary"]["final_reproj_error"] < 0.3
    print(f"\n[f4 rolling shutter] 3000 views x 144 corners, {_card()}: global {dt_g * 1e3:.1f} ms ({rgs['summary']['n_views_used']} views, "
          f"{rgs['summary']['final_reproj_error']:.3f} px), rolling {dt_r * 1e3:.1f} ms ({rrs['summary']['final_reproj_error']:.3f} px), wall incl. H2D/D2H")


@pytest.mark.gpu
def test_gpu_python_calibrator_rolling_shutter(tmp_path):
    from openimucameracalibrator_b200 import CameraCalibrator
    model, k = CASES[4]
    s = rs_sequence(model, k, **PHYS)
    doc = _corner_file(str(tmp_path / "c.uson"), s)
    cal = CameraCalibrator("EXTENDED_UNIFIED"); cal.SetGridSize(0.0); cal.SetRollingShutter()
    assert cal.CalibrateCameraFromJson(doc)
    gs = CameraCalibrator("EXTENDED_UNIFIED"); gs.SetGridSize(0.0)
    assert gs.CalibrateCameraFromJson(doc)
    assert abs(cal.result["intrinsics"][0] - k[0]) * 4 < abs(gs.result["intrinsics"][0] - k[0])
    w, u, _ = cal.api.camcal_velocities(len(s["frame_t"]))
    assert np.abs(w).max() > 0.5


@pytest.mark.gpu
def test_gpu_tool_chain_with_rolling_shutter(tmp_path):
    """calibrate_camera --pose_shutter rolling -> pose CLI --pose_shutter rolling -> rotation CLI -> hot CLI, through the files."""
    from test_cli_formats import _args
    cfg = syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), n_frames=600, grid=(8, 6), imu_rate_hz=400.0, seed=5)
    ds = syn.make_dataset(cfg)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    cams = {}
    for shutter in ("global", "rolling"):
        out = str(tmp_path / f"cam_{shutter}")
        r = subprocess.run([CAL_CLI, "--input_corners=" + paths["input_corners"], "--camera_model_to_calibrate=EXTENDED_UNIFIED", "--save_path_calib_dataset=" + out,
                            "--pose_shutter=" + shutter], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr + r.stdout
        assert ("Rolling shutter: line delay" in r.stdout) == (shutter == "rolling")
        cams[shutter] = json.load(open(out + ".json"))
        assert os.path.exists(out + ".calibdata") and os.path.exists(out + "_final_poses.ply")
    assert set(cams["rolling"]) == set(cams["global"]) and set(cams["rolling"]["intrinsics"]) == set(cams["global"]["intrinsics"])   # same layout
    cam_json, pose_json, init_json = str(tmp_path / "cam_rolling.json"), str(tmp_path / "poses.json"), str(tmp_path / "init.json")
    r = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + cam_json, "--output_pose_dataset=" + pose_json,
                        "--pose_shutter=rolling"], capture_output=True, text=True)
    assert r.returncode == 0 and "Rolling shutter: line delay" in r.stdout, r.stderr + r.stdout
    r = subprocess.run([ROT_CLI, "--input_pose_calibration_dataset=" + pose_json, "--telemetry_json=" + paths["telemetry_json"], "--imu_rotation_init_output=" + init_json],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    pth = dict(paths, camera_calibration_json=cam_json, input_pose_dataset=pose_json, gyro_to_cam_initial_calibration=init_json)
    r = subprocess.run(_args(pth, str(tmp_path)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    res = iof.read_result_json(str(tmp_path / "result.json"))
    assert np.isfinite(res["final_reproj_error"])
    # (this short, narrow-angle sequence does not pin the EXTENDED_UNIFIED focal length against alpha: the CPU oracle's composed automatic mode
    # lands on the same large-f, large-alpha fit, so the chain is checked for its files, not for the truth)
    print(f"\n[rs camcal tool chain] camera calibration error: global {cams['global']['final_reproj_error']:.4f} px, rolling "
          f"{cams['rolling']['final_reproj_error']:.4f} px; hot CLI reprojection error {res['final_reproj_error']:.4f} px")
