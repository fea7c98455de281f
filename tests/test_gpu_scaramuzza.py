"""SCARAMUZZA (Scaramuzza's omnidirectional polynomial model, OCamCalib) on the GPU: evaluation parity with the oracle on both evaluation
paths and in multi-chunk runs of its persistent-kernel instantiation, the spline LM against the oracle and the truth (pixel and tangent
error, corners past 90 degrees), the pose step's tangent error on views the normalised error loses, and the camera calibration (global and
rolling shutter, the internal initialiser, the calibrate_camera -> hot CLI and ocamcalib_to_json -> hot CLI chains).  The oracle with this
model is tests/scaramuzza/scaramuzza_oracle.cpp."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_calibration import TIGHT, H, W, _api, _qdiff, scene
from test_cli_formats import CAL_CLI, _args, _write_corner_file
from test_gpu_parity import _assert_eval_parity, _pair
from test_gpu_tmem_runs import MATRIX_FLAGS, _parity as _runs_parity, tmem_runs  # noqa: F401  (fixture)
from test_scaramuzza import K_A3, K_FIN, K_FISH, K_NEAR, SCARA, _centred, scara_oracle, scara_tangent_oracle, write_calib_results
from test_pose_estimation import _board
from test_rolling_shutter_camera_calibration import LINE_DELAY, _calibrate, _parity as _rs_parity, rs_scene
from test_tangent_spline import _parity as _tangent_parity, tangent_gpu
from test_wide_angle_poses import _view

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVAL_FLAGS = (F_STAGE1, F_ALL, F_STAGE2, capi.FLAG_T_I_C, capi.FLAG_SPLINE | capi.FLAG_GYR_BIAS, capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS,
              F_STAGE1 | capi.FLAG_GRAVITY_DIR, F_STAGE1 | capi.FLAG_CAM_INTRINSICS, F_ALL | capi.FLAG_CAM_INTRINSICS, capi.FLAG_CAM_LINE_DELAY)


KS = [K_FISH, K_FIN]
KS_IDS = ["fisheye", "finite_rho_max"]
DP = ctypes.POINTER(ctypes.c_double)


def _tiny(k, **kw):
    return syn.tiny_config(SCARA, tuple(k), **kw)


def _rot_err_deg(q, qt):
    return np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))


# ---- evaluation parity ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_eval_parity_every_column_set(gpu_factory, k, eval_path):
    o, g = _pair(scara_oracle, gpu_factory, syn.make_dataset(_tiny(k, n_frames=20, seed=9)), known_gravity=False)
    for flags in EVAL_FLAGS:
        _assert_eval_parity(o, g, flags)
    c2 = g.evaluate(F_ALL, residuals=False, gradient=False)[0]              # cost-only kernels agree with the Jacobian kernels
    assert abs(c2 - g.evaluate(F_ALL)[0]) <= 1e-12 * abs(c2)
    # POINTS (which excludes CAM_INTRINSICS): J^T J through products with random vectors, as test_gpu_points does
    flags = F_STAGE1 | capi.FLAG_POINTS
    n = g.num_tangent(flags); npts = o.get_board_points().shape[0]
    assert n == o.num_tangent(flags) == g.num_tangent(F_STAGE1) + 3 * npts
    cg, rg, gg, _ = g.evaluate(flags)
    co, ro, go, _ = o.evaluate(flags)
    assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9
    V = np.random.default_rng(8).normal(size=(3, n))
    for a, b in zip(g.normal_matvec(flags, V), o.normal_matvec(flags, V)):
        assert rel(a, b) < 1e-9


def _ragged(k, counts, grid, seed):
    ds = dict(syn.make_dataset(_tiny(k, grid=grid, n_frames=len(counts), seed=seed)))
    C = grid[0] * grid[1]
    rng = np.random.default_rng(0)
    off, ids, uv = [0], [], []
    for f, n in enumerate(counts):
        sel = np.sort(rng.choice(C, size=n, replace=False))
        ids.append(ds["point_ids"][f * C + sel]); uv.append(ds["uv"][f * C + sel]); off.append(off[-1] + n)
    ds["corner_offsets"] = np.array(off, dtype=np.int32); ds["point_ids"] = np.concatenate(ids).astype(np.int32); ds["uv"] = np.concatenate(uv)
    return ds


def test_eval_parity_ragged_frames(gpu_factory, eval_path):
    counts = [0, 1, 33, 45, 7, 32, 31, 45, 2, 45, 45, 40, 45, 45, 3, 45]
    o, g = _pair(scara_oracle, gpu_factory, _ragged(K_FISH, counts, (9, 5), 3), known_gravity=False)
    assert g.num_residuals()[0] == 2 * sum(counts)
    _assert_eval_parity(o, g, F_ALL)
    _assert_eval_parity(o, g, F_STAGE1 | capi.FLAG_CAM_INTRINSICS)


@pytest.mark.parametrize("k", [K_FIN, K_A3], ids=["finite_rho_max", "cubic"])                  # (K_FISH sees all but the negative axis)
def test_corners_outside_the_domain_give_constant_residuals(gpu_factory, k, eval_path):
    ds = dict(syn.make_dataset(_tiny(k, seed=5)))
    board = ds["board_xyzw"].copy(); board[3, :3] = [0.0, 0.0, 50.0]        # straight behind the camera: outside the domain
    ds["board_xyzw"] = board
    o, g = _pair(scara_oracle, gpu_factory, ds)
    co, ro, go, _ = o.evaluate(F_STAGE1)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    assert (ro == 1e10).sum() == (rg == 1e10).sum() == 2 * len(ds["frame_t"])
    assert np.array_equal(ro == 1e10, rg == 1e10)
    assert abs(cg - co) <= 1e-12 * co and rel(gg, go) < 1e-9


# ---- multi-chunk runs of eval_tmem_kernel<CAM_SCARAMUZZA> -----------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_multi_chunk_runs(gpu_factory, tmem_runs, k):  # noqa: F811
    seen = _runs_parity(scara_oracle, gpu_factory, tmem_runs, syn.make_dataset(_tiny(k, seed=3)), (1, 7, 13),
                        MATRIX_FLAGS + (F_STAGE1 | capi.FLAG_CAM_INTRINSICS,), known_gravity=False)
    assert {"carry", "straddle"} <= seen["vision"] | seen["imu"]


def test_ragged_frames_in_multi_chunk_runs(gpu_factory, tmem_runs):  # noqa: F811
    counts = [0, 1, 2, 3, 4, 5, 31, 32, 33, 36, 63, 64, 65, 1, 3, 2, 1, 2, 3, 65, 0, 64, 33, 5]
    seen = _runs_parity(scara_oracle, gpu_factory, tmem_runs, _ragged(K_FISH, counts, (13, 5), 17), (1, 5, 7), (F_ALL, F_STAGE2), known_gravity=False)
    assert {"carry", "straddle", "restage"} <= seen["vision"], seen


# ---- spline LM ----------------------------------------------------------------------------------------------------------------------
def test_lm_matches_the_oracle(gpu_factory):
    o, g = _pair(scara_oracle, gpu_factory, syn.make_dataset(_tiny(K_FISH, n_frames=40, seed=21, line_delay_init_scale=1.1)))
    for flags in (F_STAGE1, F_STAGE2):
        so, sg = o.optimize(30, flags), g.optimize(30, flags)
        assert sg.iterations == so.iterations and abs(sg.final_cost - so.final_cost) <= 1e-8 * so.final_cost
        assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8
    assert abs(g.get_line_delay() - o.get_line_delay()) <= 1e-8 * abs(o.get_line_delay())


def _noise_free(k, **kw):
    return syn.make_dataset(_tiny(k, n_frames=40, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0, **kw))


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_lm_recovers_the_truth(gpu_factory, k):
    ds = _noise_free(k)
    g = gpu_factory(); capi.load_dataset(g, ds)
    qt = ds["truth"]["T_i_c"]
    assert _rot_err_deg(g.get_T_i_c(), qt) > 0.5
    s = g.optimize(50, F_STAGE1)
    T = g.get_T_i_c()
    # noise-free corners, but a trajectory that no quintic B-spline holds exactly
    assert _rot_err_deg(T, qt) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-5
    assert s.mean_reproj_error < 1e-3


def _wide_dataset(k, tilt_deg=88.0, n_frames=40, seed=5):
    """A noise-free sequence of the tiny configuration with the camera tilted `tilt_deg` away from the board, so that many corners lie past
    90 degrees off the optical axis (the construction of test_tangent_spline.wide_dataset, for this model)."""
    cfg = _tiny(k, n_frames=n_frames, grid=(8, 6), seed=seed, corner_noise_px=0.0, imu_noise=False, square_m=0.05, pose_noise_m=0.0, pose_noise_rad=0.0)
    ds = syn.make_dataset(cfg)
    tilt = syn.so3_exp(np.radians(tilt_deg) * np.array([1.0, 0.0, 0.0]))
    rng = np.random.default_rng(cfg.seed)
    q_ic, t_ic = ds["truth"]["T_i_c"][:4], ds["truth"]["T_i_c"][4:]
    R_ic = syn.quat_xyzw_to_matrix(q_ic)
    R_wc_base = np.diag([1.0, -1.0, -1.0]); p_wc_base = np.array([0.0, 0.0, 0.5])
    R_wi_base = R_wc_base @ R_ic.T; p_wi_base = p_wc_base - R_wi_base @ t_ic
    traj = syn.Trajectory(rng, R_wi_base, p_wi_base)
    R_ic2 = R_ic @ tilt
    X = ds["board_xyzw"][:, :3]; C = X.shape[0]; ld = ds["truth"]["line_delay"]
    y_row = np.full((n_frames, C), H / 2.0)
    for _ in range(30):
        t_obs = ds["frame_t"][:, None] + y_row * ld * cfg.dt_so3_s
        R = traj.R_wi(t_obs.ravel()).reshape(n_frames, C, 3, 3); p = traj.p_wi(t_obs.ravel()).reshape(n_frames, C, 3)
        pcam = np.einsum("ji,fcj->fci", R_ic2, np.einsum("fcji,fcj->fci", R, X[None] - p) - t_ic)
        uv, valid = cm.project(SCARA, k, pcam)
        y_row = uv[..., 1]
    assert valid.all()
    ang = np.degrees(np.arccos(pcam[..., 2] / np.linalg.norm(pcam, axis=-1)))
    R_wc = traj.R_wi(ds["frame_t"]) @ R_ic2
    p_wc = traj.p_wi(ds["frame_t"]) + traj.R_wi(ds["frame_t"]) @ t_ic
    T_init = ds["T_i_c_init"].copy(); T_init[:4] = syn.matrix_to_quat_xyzw((syn.quat_xyzw_to_matrix(T_init[:4]) @ tilt)[None])[0]
    q2 = syn.matrix_to_quat_xyzw(R_ic2[None])[0]
    return dict(ds, uv=uv.reshape(-1, 2).copy(), q_wc=syn.matrix_to_quat_xyzw(R_wc), p_wc=p_wc, T_i_c_init=T_init, std_so3=1e-3, std_r3=1e-2,
                truth=dict(ds["truth"], T_i_c=np.concatenate([q2, t_ic]))), ang.ravel()


def test_tangent_lm_recovers_the_truth_past_90_degrees(gpu_factory):
    ds, ang = _wide_dataset(K_FISH)
    assert (ang > 90.0).sum() > 0.2 * ang.size
    g = tangent_gpu(gpu_factory, ds)
    r = g.evaluate(F_STAGE1)[1][: 2 * ang.size].reshape(-1, 2)
    assert np.isfinite(r).all() and (np.abs(r[ang > 90.0]) < 1e3).all()    # every corner past 90 degrees has a bearing and a residual
    qt = ds["truth"]["T_i_c"]
    assert _rot_err_deg(g.get_T_i_c(), qt) > 0.5
    g.optimize(50, F_STAGE1); g.optimize(10, F_STAGE2)
    T = g.get_T_i_c()
    assert _rot_err_deg(T, qt) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-6
    assert abs(g.get_line_delay() - ds["truth"]["line_delay"]) < 1e-4 * ds["truth"]["line_delay"]
    assert g.mean_reprojection_error() < 1e-4


def _numpy_bearings(k, uv):
    """unit rays of pixels, independently of the product: the stretch inverted, then the ray (u', v', F(rho))"""
    det = k[1] - k[8] * k[2]
    du, dv = uv[:, 0] - k[3], uv[:, 1] - k[4]
    up, vp = (k[1] * du - k[2] * dv) / det, (dv - k[8] * du) / det
    xyz = np.stack([up, vp, cm.scaramuzza_F(k, np.hypot(up, vp))], -1)
    xyz /= np.linalg.norm(xyz, axis=1, keepdims=True)
    px, valid = cm.project(SCARA, k, xyz)
    return xyz, (valid & (np.linalg.norm(px - uv, axis=1) < 1e-6)).astype(np.int32)


def test_tangent_evaluation_matches_the_oracle(gpu_factory):
    """the tangent oracle scores NumPy bearings of this model and the scale a0 sqrt(|c - d e|); the product forms its own"""
    ds = syn.make_dataset(_tiny(K_FISH, seed=4))
    g = tangent_gpu(gpu_factory, ds)
    o = scara_tangent_oracle(); capi.load_dataset(o, ds)
    b, ok = _numpy_bearings(K_FISH, ds["uv"])
    assert ok.all()
    b = np.ascontiguousarray(b)
    o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], len(ok), b.ctypes.data_as(DP),
            ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), K_FISH[0] * np.sqrt(abs(K_FISH[1] - K_FISH[8] * K_FISH[2])))
    for flags in (F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_TIME_OFFSET | capi.FLAG_IMU_BIASES | capi.FLAG_GRAVITY_DIR):
        _tangent_parity(g, o, flags)


# ---- pose step ------------------------------------------------------------------------------------------------------------------------
def _wide_views(k, seed, ang, front_max=None, n=3):
    """views of the pose tests' board whose centre lies `ang` degrees off the axis; with front_max, views with at most that many corners
    in front of the camera (z > 0) -> (q_wc, p_wc, uv) lists"""
    rng = np.random.default_rng(seed)
    board = _board()
    out = []
    while len(out) < n:
        v = _view(rng, SCARA, k, board, ang, dist=(0.3, 0.35), tilt=0.2) if front_max is not None else _view(rng, SCARA, k, board, ang)
        if v is None:
            continue
        pc = (board[:, :3] - v[1]) @ syn.quat_xyzw_to_matrix(v[0])
        if front_max is not None and (pc[:, 2] > 0).sum() > front_max:
            continue
        out.append(v)
    return board, out


def test_pose_step_tangent_error_keeps_views_past_90_degrees(gpu_factory):
    board, near = _wide_views(K_FISH, 1, (40.0, 60.0))
    _, far = _wide_views(K_FISH, 2, (108.0, 112.0), front_max=5)
    views = near + far
    C = board.shape[0]
    off = (np.arange(len(views) + 1) * C).astype(np.int32); ids = np.tile(np.arange(C, dtype=np.int32), len(views))
    uv = np.concatenate([v[2] for v in views]); q_true = np.array([v[0] for v in views]); p_true = np.array([v[1] for v in views])
    g = gpu_factory(); g.set_camera(SCARA, K_FISH, W, H); g.set_board_points(board)
    v_norm = g.estimate_board_poses(off, ids, uv)[3]
    assert v_norm[:3].all() and not v_norm[3:].any()                        # the normalised error cannot place them
    g = gpu_factory(); g.set_camera(SCARA, K_FISH, W, H); g.set_board_points(board); g.set_pose_error("tangent")
    q, p, e, v = g.estimate_board_poses(off, ids, uv)
    assert v.all()
    assert _qdiff(q, q_true).max() < 1e-8 and np.abs(p - p_true).max() < 1e-8 and e.max() < 1e-8


# ---- camera calibration ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_calibration_matches_the_oracle(gpu_factory, k):
    B, off, ids, uv, q_true, p_true = scene(SCARA, k, n_views=36, seed=47, noise_px=0.2)
    uv[off[5] + 7] += 25.0                                                   # a gross outlier inside the Huber tail
    ro = _api(scara_oracle, B).calibrate_camera(SCARA, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    rg = _api(gpu_factory, B).calibrate_camera(SCARA, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    so, sg = ro["summary"], rg["summary"]
    assert sg["success"] == 1 and so["success"] == 1 and (rg["used"] == ro["used"]).all() and sg["gpu_launches"] > 0
    assert abs(sg["focal_length_init"] - so["focal_length_init"]) < 1e-4 * so["focal_length_init"]
    assert ro["intrinsics"][2] != 0.0 and ro["intrinsics"][8] != 0.0        # stage 3 frees the stretch e, d
    # the antisymmetric part of the stretch (e = -d) is, to first order, a turn of the sensor about the optical axis that the view poses
    # absorb, so the two solvers may settle anywhere along that shallow valley: compare what the calibration predicts, not (e, d, c, poses)
    assert np.abs(rg["intrinsics"][[0, 3, 4, 5, 6, 7]] - ro["intrinsics"][[0, 3, 4, 5, 6, 7]]).max() / ro["intrinsics"][0] < 1e-6
    for v in np.flatnonzero(ro["used"]):
        X = B[ids[off[v]:off[v + 1]], :3]
        pg = cm.project(SCARA, rg["intrinsics"], (X - rg["p_wc"][v]) @ syn.quat_xyzw_to_matrix(rg["q_wc"][v]))[0]
        po = cm.project(SCARA, ro["intrinsics"], (X - ro["p_wc"][v]) @ syn.quat_xyzw_to_matrix(ro["q_wc"][v]))[0]
        assert np.abs(pg - po).max() < 1e-3                                  # px
    assert np.abs(rg["view_error_px"] - ro["view_error_px"]).max() < 1e-6
    assert abs(sg["final_cost"][2] - so["final_cost"][2]) < 1e-7 * so["final_cost"][2]


@pytest.mark.parametrize("k", [K_NEAR, K_FISH], ids=["near_pinhole", "fisheye"])
def test_internal_initialiser_recovers_the_truth(gpu_factory, k):
    k = _centred(k)
    B, off, ids, uv, q_true, p_true = scene(SCARA, k, seed=3)
    r = _api(gpu_factory, B).calibrate_camera(SCARA, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and s["n_views_used"] == 30 and r["used"].all()
    px, _ = cm.project(SCARA, r["intrinsics"], _view_rays())
    assert np.abs(px - cm.project(SCARA, k, _view_rays())[0]).max() < 1e-6     # the same camera
    assert np.abs(r["intrinsics"][:5] - k[:5]).max() < 1e-6 * k[0]
    assert _qdiff(r["q_wc"], q_true).max() < 1e-8 and np.abs(r["p_wc"] - p_true).max() < 1e-8


def _view_rays():
    th = np.radians(np.linspace(0.0, 60.0, 50)); ph = np.linspace(0.0, 2 * np.pi, 50)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


def test_rolling_shutter_calibration_fixed_mode_matches_the_oracle(gpu_factory):
    B, off, ids, uv, vel = rs_scene(SCARA, K_FISH, n_views=36, seed=67)
    uv[off[5] + 7] += 25.0
    s = dict(board=B, off=off, ids=ids, uv=uv)
    o, g = scara_oracle(), gpu_factory()
    for a in (o, g):
        a.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    _rs_parity(_calibrate(g, SCARA, s), _calibrate(o, SCARA, s), SCARA)


def test_calibrate_camera_cli_output_feeds_the_hot_cli(tmp_path):
    k = _centred(K_FISH)
    B, off, ids, uv, q_true, p_true = scene(SCARA, k, n_views=40, seed=17, noise_px=0.1)
    corners = str(tmp_path / "corners.uson")
    _write_corner_file(corners, B, off, ids, uv)
    out = subprocess.run([CAL_CLI, "--input_corners=" + corners, "--camera_model_to_calibrate=SCARAMUZZA", "--save_path_calib_dataset=" + str(tmp_path / "cam"),
                          "--grid_size=0.001"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "SCARAMUZZA model: A2: " in out.stdout
    cam = json.load(open(str(tmp_path / "cam.json")))
    assert cam["intrinsic_type"] == "SCARAMUZZA"
    i = cam["intrinsics"]
    got = np.array([i["focal_length"], i["aspect_ratio"], i["stretch_e"], i["principal_pt_x"], i["principal_pt_y"], i["polynomial_a2"], i["polynomial_a3"],
                    i["polynomial_a4"], i["stretch_d"]])
    assert cam["final_reproj_error"] < 0.2                                # 0.1 px noise
    # the hot CLI reads that calibration next to a sequence of its own
    paths = iof.write_dataset_files(syn.make_dataset(_tiny(K_FISH, n_frames=8)), str(tmp_path / "seq"))
    paths["camera_calibration_json"] = str(tmp_path / "cam.json")
    out = subprocess.run(_args(paths, str(tmp_path), ["--parse_only"]), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == 8 and np.allclose(s["intrinsics"], got, rtol=1e-12, atol=0)


def test_ocamcalib_import_feeds_the_hot_cli(tmp_path):
    """calib_results.txt -> ocamcalib_to_json -> a spline solve of the hot CLI on a sequence projected through the imported camera"""
    src, cam = str(tmp_path / "calib_results.txt"), str(tmp_path / "cam.json")
    write_calib_results(src)
    out = subprocess.run([sys.executable, "-m", "openimucameracalibrator_b200.ocamcalib_to_json", "--input", src, "--output", cam, "--fps", "30"],
                         capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    i = json.load(open(cam))["intrinsics"]
    k = np.array([i["focal_length"], i["aspect_ratio"], i["stretch_e"], i["principal_pt_x"], i["principal_pt_y"], i["polynomial_a2"], i["polynomial_a3"],
                  i["polynomial_a4"], i["stretch_d"]])
    ds = syn.make_dataset(_tiny(k, n_frames=30, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
    paths = iof.write_dataset_files(ds, str(tmp_path / "seq"))
    paths["camera_calibration_json"] = cam
    out = subprocess.run(_args(paths, str(tmp_path), []), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr + out.stdout
    res = json.load(open(str(tmp_path / "result.json")))
    assert res
