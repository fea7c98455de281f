"""FISHEYE_RADIAL_TANGENTIAL (Kannala-Brandt with k1..k6 and tangential t1, t2) on the GPU: evaluation parity with the oracle on both
evaluation paths, in multi-chunk runs of its persistent-kernel instantiation, in tangent mode and with POINTS; the three intrinsic columns past
the oracle's ten against central differences of the GPU cost; corners outside the domain; the reduction to FISHEYE; the spline LM against the
oracle and the truth; the pose step; the camera calibration (global and rolling shutter); BASELINE config 4's size; and the tool chain
calibrate_camera -> pose CLI -> rotation CLI -> hot CLI.  The oracle is tests/fisheye_radtan/fisheye_radtan_oracle.cpp: the unchanged CPU
oracle with the model added, its k6, t1, t2 held constant."""
import ctypes
import dataclasses
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_calibration import TIGHT, H, W, _api, _qdiff, scene
from test_cli_formats import CAL_CLI, POSE_CLI, ROT_CLI, _args
from test_fisheye_radtan import FR, K_SKEW, K_WIDE
from test_gpu_parity import _assert_eval_parity
from test_gpu_tmem_runs import MATRIX_FLAGS, _parity as _runs_parity, tmem_runs  # noqa: F401  (fixture)
from test_rolling_shutter_camera_calibration import LINE_DELAY, _calibrate, rs_scene
from test_tangent_spline import _parity as _tangent_parity, tangent_gpu

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DP = ctypes.POINTER(ctypes.c_double)
EVAL_FLAGS = (F_STAGE1, F_ALL, F_STAGE2, capi.FLAG_T_I_C, capi.FLAG_SPLINE | capi.FLAG_GYR_BIAS, capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS,
              F_STAGE1 | capi.FLAG_GRAVITY_DIR, capi.FLAG_CAM_LINE_DELAY, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_TIME_OFFSET)
KS, KS_IDS = [K_WIDE, K_SKEW], ["wide", "skew"]
# a wide lens centred in the image, for the camera calibration (RunCalibration's schedule pins the principal point in stage 1), and the
# same lens decentred
K_CAL = np.array([300.0, 1.0, 0.0, W / 2, H / 2, 0.04, -0.01, 0.002, -3e-4, 2e-5, -1e-6, 0.0, 0.0])
K_DEC = np.concatenate([K_CAL[:11], [1.5e-3, -1e-3]])

_LIBS = {}


def _oracle_lib(tangent=False):
    if tangent not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_fisheye_radtan_oracle_"), "libfisheye_radtan_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + (["-DFISHEYE_RADTAN_TANGENT"] if tangent else []) +
                              ["-o", out, os.path.join(HERE, "fisheye_radtan", "fisheye_radtan_oracle.cpp")])
        _LIBS[tangent] = ctypes.CDLL(out)
    return _LIBS[tangent]


def _set_tail(lib, k):
    lib.fisheye_radtan_oracle_set_tail(np.ascontiguousarray(np.asarray(k)[10:13], dtype=np.float64).ctypes.data_as(DP))


def fr_oracle(ds, tangent=False, **kw):
    """the oracle on `ds`: its first ten intrinsics as the camera, k6, t1, t2 held constant"""
    lib = _oracle_lib(tangent)
    _set_tail(lib, ds["intrinsics"])
    o = capi.CApi(lib, "icco_", 0)
    d = dict(ds); d["intrinsics"] = np.asarray(ds["intrinsics"])[:10]
    capi.load_dataset(o, d, **kw)
    return o


class _TruncatingOracle:
    """the oracle's CApi, handed the first ten intrinsics by whoever sets the camera"""
    def __init__(self, api):
        self._api = api

    def set_camera(self, model, intr, w, h):
        return self._api.set_camera(model, np.asarray(intr)[:10], w, h)

    def __getattr__(self, name):
        return getattr(self._api, name)


def _tiny(k, **kw):
    return syn.tiny_config(FR, tuple(k), **kw)


def _pair(gpu_factory, ds, **kw):
    g = gpu_factory(); capi.load_dataset(g, ds, **kw)
    return fr_oracle(ds, **kw), g


def _rot_err_deg(q, qt):
    return np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))


# ---- evaluation parity ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_eval_parity_every_column_set(gpu_factory, k, eval_path):
    o, g = _pair(gpu_factory, syn.make_dataset(_tiny(k, n_frames=20, seed=9)), known_gravity=False)
    for flags in EVAL_FLAGS:
        _assert_eval_parity(o, g, flags)
    flags = F_STAGE1 | capi.FLAG_POINTS
    n = g.num_tangent(flags)
    assert n == o.num_tangent(flags)
    cg, rg, gg, _ = g.evaluate(flags)
    co, ro, go, _ = o.evaluate(flags)
    assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9
    V = np.random.default_rng(8).normal(size=(3, n))
    for a, b in zip(g.normal_matvec(flags, V), o.normal_matvec(flags, V)):
        assert rel(a, b) < 1e-9


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_thirteen_intrinsic_columns(gpu_factory, k, eval_path):
    """CAM_INTRINSICS: the first ten columns against the oracle's ten, k6, t1, t2 against central differences of the GPU residuals"""
    ds = syn.make_dataset(_tiny(k, n_frames=20, seed=11))
    o, g = _pair(gpu_factory, ds)
    for flags in (F_STAGE1 | capi.FLAG_CAM_INTRINSICS, F_ALL | capi.FLAG_CAM_INTRINSICS):
        n = g.num_tangent(flags)
        assert n == o.num_tangent(flags) + 3
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        co, ro, go, Ho = o.evaluate(flags, hessian=True)
        last = n - 3
        assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg[:last], go) < 1e-9 and rel(Hg[:last, :last], Ho) < 1e-9
        assert np.array_equal(Hg, Hg.T) and np.abs(Hg[last:, last:]).min() > 0.0
    n = g.num_tangent(F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    _, r0, gg, _ = g.evaluate(F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    # the gradient entry r . dr/dk_j, dr/dk_j by central differences of the residuals: they are quadratic in k6 (theta_d is linear in it, the
    # tangential stage quadratic in theta_d) and linear in t1, t2, so a step as large as 1e-3 is exact up to rounding and keeps the
    # residuals' changes far above it
    for j in range(3):
        h = 1e-3
        res = []
        for sgn in (1.0, -1.0):
            d = dict(ds); kk = np.array(ds["intrinsics"], dtype=np.float64); kk[10 + j] += sgn * h; d["intrinsics"] = kk
            a = gpu_factory(); capi.load_dataset(a, d)
            res.append(a.evaluate(F_STAGE1, gradient=False)[1])
        fd = float(r0 @ ((res[0] - res[1]) / (2 * h)))
        assert abs(fd - gg[n - 3 + j]) <= 1e-5 * abs(gg[n - 3 + j]), (j, fd, gg[n - 3 + j])


def test_reduced_model_equals_fisheye(gpu_factory, eval_path):
    k = K_SKEW.copy(); k[9:] = 0.0
    ds = syn.make_dataset(_tiny(k, n_frames=20, seed=5))
    d9 = dict(ds); d9["model"] = cm.FISHEYE; d9["intrinsics"] = k[:9]
    g = gpu_factory(); capi.load_dataset(g, ds)
    f = gpu_factory(); capi.load_dataset(f, d9)
    for flags in (F_ALL, F_STAGE1 | capi.FLAG_CAM_INTRINSICS):
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        cf, rf, gf, Hf = f.evaluate(flags, hessian=True)
        m = gf.size
        assert abs(cg - cf) <= 1e-12 * cf and rel(rg, rf) < 1e-12 and rel(gg[:m], gf) < 1e-12 and rel(Hg[:m, :m], Hf) < 1e-12


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_corners_behind_the_camera_give_constant_residuals(gpu_factory, k, eval_path):
    ds = dict(syn.make_dataset(_tiny(k, seed=5)))
    board = ds["board_xyzw"].copy(); board[3, :3] = [0.0, 0.0, 50.0]        # behind the camera: z <= 0
    ds["board_xyzw"] = board
    o, g = _pair(gpu_factory, ds)
    co, ro, go, _ = o.evaluate(F_STAGE1)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    assert (ro == 1e10).sum() == (rg == 1e10).sum() >= 2 * len(ds["frame_t"])
    assert np.array_equal(ro == 1e10, rg == 1e10)
    assert abs(cg - co) <= 1e-12 * co and rel(gg, go) < 1e-9


def test_corners_past_the_fold_give_constant_residuals(gpu_factory, eval_path):
    """a k1 that folds theta_d inside the field of the sequence: the corners beyond theta_max fail on the device and in the oracle alike"""
    ds = syn.make_dataset(_tiny(K_WIDE, n_frames=20, seed=13))
    xy, ok = cm.fisheye_radtan_unproject(K_WIDE, ds["uv"])
    th = np.arctan(np.hypot(xy[:, 0], xy[:, 1]))
    for k1 in np.linspace(-0.5, -20.0, 80):                                # theta_max = sqrt(-1 / (3 k1)) for k1 alone
        k = K_WIDE.copy(); k[5] = k1
        if 0.05 < (th >= cm.fisheye_radtan_theta_max(k)).mean() < 0.95:
            break
    else:
        pytest.fail("no k1 folds inside the sequence's field")
    d = dict(ds); d["intrinsics"] = k
    o, g = _pair(gpu_factory, d)
    co, ro, _, _ = o.evaluate(F_STAGE1)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    assert (rg == 1e10).any() and np.array_equal(ro == 1e10, rg == 1e10) and abs(cg - co) <= 1e-12 * co


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_multi_chunk_runs(gpu_factory, tmem_runs, k):  # noqa: F811
    ds = syn.make_dataset(_tiny(k, seed=3))

    def oracle():
        lib = _oracle_lib(); _set_tail(lib, ds["intrinsics"])
        return _TruncatingOracle(capi.CApi(lib, "icco_", 0))
    seen = _runs_parity(oracle, gpu_factory, tmem_runs, ds, (1, 7, 13), MATRIX_FLAGS, known_gravity=False)
    assert {"carry", "straddle"} <= seen["vision"] | seen["imu"]


def test_tangent_evaluation_matches_the_oracle(gpu_factory):
    """the tangent oracle scores NumPy bearings of this model at the scale f sqrt(ar); the product forms its own"""
    ds = syn.make_dataset(_tiny(K_WIDE, seed=4))
    g = tangent_gpu(gpu_factory, ds)
    o = fr_oracle(ds, tangent=True)
    xy, ok = cm.fisheye_radtan_unproject(K_WIDE, ds["uv"])
    assert ok.all()
    b = np.concatenate([xy, np.ones((xy.shape[0], 1))], 1)
    b = np.ascontiguousarray(b / np.linalg.norm(b, axis=1, keepdims=True))
    ok = ok.astype(np.int32)
    o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], len(ok), b.ctypes.data_as(DP),
            ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), K_WIDE[0] * np.sqrt(K_WIDE[1]))
    for flags in (F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_TIME_OFFSET | capi.FLAG_IMU_BIASES | capi.FLAG_GRAVITY_DIR):
        _tangent_parity(g, o, flags)


# ---- spline LM ----------------------------------------------------------------------------------------------------------------------
def test_lm_matches_the_oracle(gpu_factory):
    o, g = _pair(gpu_factory, syn.make_dataset(_tiny(K_WIDE, n_frames=40, seed=21, line_delay_init_scale=1.1)))
    for flags in (F_STAGE1, F_STAGE2):
        so, sg = o.optimize(30, flags), g.optimize(30, flags)
        assert sg.iterations == so.iterations
        assert abs(sg.final_cost - so.final_cost) <= 1e-7 * so.final_cost
        assert np.abs(g.get_T_i_c() - o.get_T_i_c()).max() < 1e-7
        assert abs(g.get_line_delay() - o.get_line_delay()) < 1e-7 * abs(o.get_line_delay())


def test_lm_recovers_the_truth_on_a_decentred_lens(gpu_factory):
    k = K_WIDE.copy(); k[11:] = (4e-3, -3e-3)                                 # a lens well off-centre in its mount
    ds = syn.make_dataset(_tiny(k, n_frames=40, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
    g = gpu_factory(); capi.load_dataset(g, ds)
    qt = ds["truth"]["T_i_c"]
    assert _rot_err_deg(g.get_T_i_c(), qt) > 0.5
    g.optimize(50, F_STAGE1)
    T = g.get_T_i_c()
    assert _rot_err_deg(T, qt) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-5
    assert g.mean_reprojection_error() < 1e-3


# ---- pose step ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["normalized", "tangent"])
def test_pose_step_recovers_the_poses(gpu_factory, mode):
    B, off, ids, uv, q_true, p_true = scene(FR, K_CAL, n_views=12, seed=31)
    g = gpu_factory(); g.set_camera(FR, K_CAL, W, H); g.set_board_points(B); g.set_pose_error(mode)
    q, p, e, v = g.estimate_board_poses(off, ids, uv)
    assert v.all() and _qdiff(q, q_true).max() < 1e-8 and np.abs(p - p_true).max() < 1e-8 and e.max() < 1e-8


@pytest.mark.parametrize("mode", ["normalized", "tangent"])
def test_rolling_shutter_pose_step(gpu_factory, mode):
    """the rolling-shutter pose passes take the corners at their row times: every view keeps its pose, and the poses move off the global
    shutter's"""
    B, off, ids, uv, vel = rs_scene(FR, K_CAL, n_views=12, seed=67)
    frame_t = np.arange(12) * 0.05
    res = {}
    for ld in (0.0, LINE_DELAY):
        g = gpu_factory(); g.set_camera(FR, K_CAL, W, H); g.set_board_points(B); g.set_pose_error(mode)
        g.set_pose_rolling_shutter(ld, frame_t if ld > 0 else None)
        res[ld] = g.estimate_board_poses(off, ids, uv)
        assert res[ld][3].all()
    assert np.isfinite(res[LINE_DELAY][0]).all() and np.abs(res[LINE_DELAY][1] - res[0.0][1]).max() > 0.0


# ---- camera calibration ---------------------------------------------------------------------------------------------------------------
def _rays(uv):
    """rays over the field the views cover: out to the widest corner's angle (six radial terms are not held to anything beyond it)"""
    xy, ok = cm.fisheye_radtan_unproject(K_CAL, uv)
    assert ok.all()
    th = np.linspace(0.0, np.arctan(np.hypot(xy[:, 0], xy[:, 1]).max()), 60); ph = np.linspace(0.0, 2 * np.pi, 60)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


def test_calibration_recovers_the_camera(gpu_factory):
    B, off, ids, uv, q_true, p_true = scene(FR, K_CAL, n_views=36, seed=3)
    r = _api(gpu_factory, B).calibrate_camera(FR, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and r["used"].all() and r["intrinsics"].size == 13
    assert np.abs(r["intrinsics"][11:]).max() < 1e-7                          # stage 3 frees t1, t2
    px = cm.project(FR, r["intrinsics"], _rays(uv))[0]
    assert np.abs(px - cm.project(FR, K_CAL, _rays(uv))[0]).max() < 1e-3     # the same camera over the calibrated field
    assert np.abs(r["intrinsics"][[0, 3, 4]] - K_CAL[[0, 3, 4]]).max() < 1e-4 * K_CAL[0]
    assert _qdiff(r["q_wc"], q_true).max() < 1e-6 and np.abs(r["p_wc"] - p_true).max() < 1e-6 and s["final_reproj_error"] < 1e-5


def test_calibration_recovers_a_decentred_lens(gpu_factory):
    """a lens with t1, t2 != 0: stage 3 frees them and they come back near the truth, and the fit is far closer than FISHEYE's on the same
    corners.  Noise-free, it stops at about 0.01 px rather than 0: stage 1 fits k1..k6 without the tangential terms, and from there the
    six-term radial polynomial (theta^3 .. theta^13 are nearly collinear over the field) leaves the normal equations too ill-conditioned for
    the last steps of stage 3 to be accepted."""
    B, off, ids, uv, q_true, p_true = scene(FR, K_DEC, n_views=36, seed=3)
    r = _api(gpu_factory, B).calibrate_camera(FR, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and r["used"].all()
    t = r["intrinsics"][11:]
    assert (np.abs(t - K_DEC[11:]) < 0.2 * np.abs(K_DEC[11:])).all(), t
    assert np.abs(cm.project(FR, r["intrinsics"], _rays(uv))[0] - cm.project(FR, K_DEC, _rays(uv))[0]).max() < 1.0
    rf = _api(gpu_factory, B).calibrate_camera(cm.FISHEYE, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    print(f"\n[decentred lens] FISHEYE_RADIAL_TANGENTIAL {s['final_reproj_error']:.4f} px (t1, t2 = {t[0]:.3e}, {t[1]:.3e}), "
          f"FISHEYE {rf['summary']['final_reproj_error']:.4f} px")
    assert s["final_reproj_error"] < 0.02 and s["final_reproj_error"] < 0.5 * rf["summary"]["final_reproj_error"]


def test_rolling_shutter_calibration_recovers_the_camera(gpu_factory):
    B, off, ids, uv, vel = rs_scene(FR, K_CAL, n_views=36, seed=67, noise_px=0.0)
    g = gpu_factory(); g.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    r = _calibrate(g, FR, dict(board=B, off=off, ids=ids, uv=uv))
    assert r["summary"]["success"] == 1 and r["used"].all()
    assert np.abs(cm.project(FR, r["intrinsics"], _rays(uv))[0] - cm.project(FR, K_CAL, _rays(uv))[0]).max() < 1e-3


# ---- full size ------------------------------------------------------------------------------------------------------------------------
def test_config4_size_lm_iteration_and_normal_matvec():
    """BASELINE config 4's sequence (3000 views x 144 corners) in this model: one full LM iteration, and J^T J products with random
    vectors equal the oracle's"""
    from openimucameracalibrator_b200 import calibrator
    k = (438.0, 1.0, 0.0, 489.5, 272.0, 0.02, -0.004, 6e-4, -5e-5, 2e-6, -3e-8, 1.2e-3, -8e-4)
    ds = syn.make_dataset(dataclasses.replace(syn.CONFIGS[4], name="cfg4_fisheye_radtan_3000x144", model=FR, intrinsics=k))
    g = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(g, ds)
    o = fr_oracle(ds)
    n = g.num_tangent(F_STAGE1)
    assert n == o.num_tangent(F_STAGE1) and g.num_residuals()[0] == 864000
    V = np.random.default_rng(44).normal(size=(3, n)); V[1, : n - 6] = 0.0; V[2, n - 6:] = 0.0
    for a, b in zip(g.normal_matvec(F_STAGE1, V), o.normal_matvec(F_STAGE1, V)):
        assert rel(a, b) < 1e-9
    s = g.lm_iterations(1, F_STAGE1)
    assert s.successful_steps == 1 and s.final_cost < s.initial_cost and np.isfinite(g.get_T_i_c()).all()


# ---- tool chain ------------------------------------------------------------------------------------------------------------------------
def test_tool_chain_calibrate_camera_pose_rotation_hot_cli(tmp_path):
    cfg = syn.tiny_config(FR, tuple(K_WIDE), n_frames=300, grid=(8, 6), imu_rate_hz=400.0, seed=5)
    ds = syn.make_dataset(cfg)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    cam = str(tmp_path / "cam")
    r = subprocess.run([CAL_CLI, "--input_corners=" + paths["input_corners"], "--camera_model_to_calibrate=FISHEYE_RADIAL_TANGENTIAL", "--save_path_calib_dataset=" + cam],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    assert "FISHEYE_RADIAL_TANGENTIAL model: Radial distortion 1: " in r.stdout and "Tangential distortion 2: " in r.stdout
    doc = json.load(open(cam + ".json"))
    assert doc["intrinsic_type"] == "FISHEYE_RADIAL_TANGENTIAL" and set(doc["intrinsics"]) == set(cm.CAMERAS[FR].keys)
    pose_json, init_json = str(tmp_path / "poses.json"), str(tmp_path / "init.json")
    r = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + cam + ".json", "--output_pose_dataset=" + pose_json],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    r = subprocess.run([ROT_CLI, "--input_pose_calibration_dataset=" + pose_json, "--telemetry_json=" + paths["telemetry_json"], "--imu_rotation_init_output=" + init_json],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    pth = dict(paths, camera_calibration_json=cam + ".json", input_pose_dataset=pose_json, gyro_to_cam_initial_calibration=init_json)
    r = subprocess.run(_args(pth, str(tmp_path)), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    res = iof.read_result_json(str(tmp_path / "result.json"))
    assert np.isfinite(res["final_reproj_error"])
    # (as in the other tool-chain tests, this short sequence is checked for its hand-overs, not for the truth)
    print(f"\n[fisheye-radtan tool chain] camera calibration error {doc['final_reproj_error']:.4f} px, hot CLI reprojection error "
          f"{res['final_reproj_error']:.4f} px")
