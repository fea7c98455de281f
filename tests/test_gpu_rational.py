"""PINHOLE_RATIONAL (OpenCV's rational polynomial model) on the GPU: evaluation parity with the oracle on both evaluation paths and in
multi-chunk runs of its persistent-kernel instantiation (pixel and tangent residuals, corners outside the domain), the three intrinsic
columns past the oracle's ten against central differences, the spline LM against the oracle and the truth, the pose step, the camera
calibration (global and rolling shutter) and the opencv_to_json / calibrate_camera -> hot CLI chains.  The oracle is
tests/rational/rational_oracle.cpp: the unchanged CPU oracle with the model added, its denominator k4..k6 held constant."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_calibration import TIGHT, H, W, _api, _qdiff, scene
from test_cli_formats import CAL_CLI, _args, _write_corner_file
from test_gpu_parity import _assert_eval_parity
from test_gpu_tmem_runs import MATRIX_FLAGS, _parity as _runs_parity, tmem_runs  # noqa: F401  (fixture)
from test_rational import K_SKEW, K_WIDE, RAT, _opencv_yaml
from test_rolling_shutter_camera_calibration import LINE_DELAY, _calibrate, rs_scene
from test_tangent_spline import _parity as _tangent_parity, tangent_gpu

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DP = ctypes.POINTER(ctypes.c_double)
EVAL_FLAGS = (F_STAGE1, F_ALL, F_STAGE2, capi.FLAG_T_I_C, capi.FLAG_SPLINE | capi.FLAG_GYR_BIAS, capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS,
              F_STAGE1 | capi.FLAG_GRAVITY_DIR, capi.FLAG_CAM_LINE_DELAY, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_TIME_OFFSET)
KS, KS_IDS = [K_WIDE, K_SKEW], ["wide", "skew"]
# a mild lens centred in the image, for the camera calibration (RunCalibration's schedule pins the principal point in stage 1)
K_CAL = np.array([420.0, 1.0, 0.0, W / 2, H / 2, 0.12, -0.03, 0.004, 0.0, 0.0, 0.06, 0.01, -0.002])

_LIBS = {}


def _oracle_lib(tangent=False):
    if tangent not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_rational_oracle_"), "librational_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + (["-DRATIONAL_TANGENT"] if tangent else []) +
                              ["-o", out, os.path.join(HERE, "rational", "rational_oracle.cpp")])
        _LIBS[tangent] = ctypes.CDLL(out)
    return _LIBS[tangent]


def rational_oracle(ds, tangent=False, **kw):
    """the oracle on `ds`: its first ten intrinsics as the camera, the denominator k4..k6 held constant"""
    lib = _oracle_lib(tangent)
    lib.rational_oracle_set_denominator(np.ascontiguousarray(ds["intrinsics"][10:13], dtype=np.float64).ctypes.data_as(DP))
    o = capi.CApi(lib, "icco_", 0)
    d = dict(ds); d["intrinsics"] = np.asarray(ds["intrinsics"])[:10]
    capi.load_dataset(o, d, **kw)
    return o


def _tiny(k, **kw):
    return syn.tiny_config(RAT, tuple(k), **kw)


def _pair(gpu_factory, ds, **kw):
    g = gpu_factory(); capi.load_dataset(g, ds, **kw)
    return rational_oracle(ds, **kw), g


def _rot_err_deg(q, qt):
    return np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))


# ---- evaluation parity ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_eval_parity_every_column_set(gpu_factory, k, eval_path):
    o, g = _pair(gpu_factory, syn.make_dataset(_tiny(k, n_frames=20, seed=9)), known_gravity=False)
    for flags in EVAL_FLAGS:
        _assert_eval_parity(o, g, flags)
    flags = F_STAGE1 | capi.FLAG_POINTS
    cg, rg, gg, _ = g.evaluate(flags)
    co, ro, go, _ = o.evaluate(flags)
    assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_thirteen_intrinsic_columns(gpu_factory, k, eval_path):
    """CAM_INTRINSICS: the first ten columns against the oracle's ten, the denominator's three against central differences of the cost"""
    ds = syn.make_dataset(_tiny(k, n_frames=20, seed=11))
    o, g = _pair(gpu_factory, ds)
    for flags in (F_STAGE1 | capi.FLAG_CAM_INTRINSICS, F_ALL | capi.FLAG_CAM_INTRINSICS):
        n = g.num_tangent(flags)
        assert n == o.num_tangent(flags) + 3
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        co, ro, go, Ho = o.evaluate(flags, hessian=True)
        last = n - 3 if flags & capi.FLAG_TIME_OFFSET == 0 else None
        assert last is not None
        assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg[:last], go) < 1e-9 and rel(Hg[:last, :last], Ho) < 1e-9
        assert np.array_equal(Hg, Hg.T) and np.abs(Hg[last:, last:]).min() > 0.0
    n = g.num_tangent(F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    _, r0, gg, _ = g.evaluate(F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    for j in range(3):                           # the gradient entry r . dr/dk_j, dr/dk_j by central differences of the residuals
        h = 1e-4 * max(abs(k[10 + j]), 1e-2)    # rounding of pixels ~500 limits smaller steps
        res = []
        for sgn in (1.0, -1.0):
            d = dict(ds); kk = np.array(ds["intrinsics"], dtype=np.float64); kk[10 + j] += sgn * h; d["intrinsics"] = kk
            a = gpu_factory(); capi.load_dataset(a, d)
            res.append(a.evaluate(F_STAGE1, gradient=False)[1])
        fd = float(r0 @ ((res[0] - res[1]) / (2 * h)))
        assert abs(fd - gg[n - 3 + j]) <= 1e-5 * abs(gg[n - 3 + j]), (j, fd, gg[n - 3 + j])


def test_zero_denominator_equals_the_radial_tangential_model(gpu_factory, eval_path):
    k = K_SKEW.copy(); k[10:] = 0.0
    ds = syn.make_dataset(_tiny(k, n_frames=20, seed=5))
    d10 = dict(ds); d10["model"] = cm.PINHOLE_RADIAL_TANGENTIAL; d10["intrinsics"] = k[:10]
    g = gpu_factory(); capi.load_dataset(g, ds)
    r = gpu_factory(); capi.load_dataset(r, d10)
    for flags in (F_ALL, F_STAGE1 | capi.FLAG_CAM_INTRINSICS):
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        cr, rr, gr, Hr = r.evaluate(flags, hessian=True)
        m = gr.size
        assert abs(cg - cr) <= 1e-12 * cr and rel(rg, rr) < 1e-12 and rel(gg[:m], gr) < 1e-12 and rel(Hg[:m, :m], Hr) < 1e-12


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_corners_outside_the_domain_give_constant_residuals(gpu_factory, k, eval_path):
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
    """a denominator that folds the lens inside the field of the sequence: the corners beyond s_max fail on the device and in the oracle alike"""
    ds = syn.make_dataset(_tiny(K_WIDE, n_frames=20, seed=13))
    xy, ok = cm.rational_unproject(K_WIDE, ds["uv"])
    s = (xy ** 2).sum(1)
    for k4 in (64.0, 128.0, 256.0):                                         # s_max = 0.016, 0.0079, 0.0039 (the corners reach s = 0.026)
        k = K_WIDE.copy(); k[10] = k4
        if 0.05 < (s >= cm.rational_s_max(k)).mean() < 0.95:
            break
    else:
        pytest.fail("no denominator folds inside the sequence's field")
    d = dict(ds); d["intrinsics"] = k
    o, g = _pair(gpu_factory, d)
    co, ro, _, _ = o.evaluate(F_STAGE1)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    assert (rg == 1e10).any() and np.array_equal(ro == 1e10, rg == 1e10) and abs(cg - co) <= 1e-12 * co


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_multi_chunk_runs(gpu_factory, tmem_runs, k):  # noqa: F811
    ds = syn.make_dataset(_tiny(k, seed=3))
    seen = _runs_parity(lambda: rational_oracle_factory(ds), gpu_factory, tmem_runs, ds, (1, 7, 13), MATRIX_FLAGS, known_gravity=False)
    assert {"carry", "straddle"} <= seen["vision"] | seen["imu"]


def rational_oracle_factory(ds):
    lib = _oracle_lib()
    lib.rational_oracle_set_denominator(np.ascontiguousarray(ds["intrinsics"][10:13], dtype=np.float64).ctypes.data_as(DP))
    return _TruncatingOracle(capi.CApi(lib, "icco_", 0))


class _TruncatingOracle:
    """the oracle's CApi, handed the first ten intrinsics by whoever sets the camera"""
    def __init__(self, api):
        self._api = api

    def set_camera(self, model, intr, w, h):
        return self._api.set_camera(model, np.asarray(intr)[:10], w, h)

    def __getattr__(self, name):
        return getattr(self._api, name)


def test_tangent_evaluation_matches_the_oracle(gpu_factory):
    """the tangent oracle scores NumPy bearings of this model at the scale f sqrt(ar); the product forms its own"""
    ds = syn.make_dataset(_tiny(K_WIDE, seed=4))
    g = tangent_gpu(gpu_factory, ds)
    o = rational_oracle(ds, tangent=True)
    xy, ok = cm.rational_unproject(K_WIDE, ds["uv"])
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


def test_lm_recovers_the_truth(gpu_factory):
    ds = syn.make_dataset(_tiny(K_WIDE, n_frames=40, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
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
    B, off, ids, uv, q_true, p_true = scene(RAT, K_CAL, n_views=12, seed=31)
    g = gpu_factory(); g.set_camera(RAT, K_CAL, W, H); g.set_board_points(B); g.set_pose_error(mode)
    q, p, e, v = g.estimate_board_poses(off, ids, uv)
    assert v.all() and _qdiff(q, q_true).max() < 1e-8 and np.abs(p - p_true).max() < 1e-8 and e.max() < 1e-8


@pytest.mark.parametrize("mode", ["normalized", "tangent"])
def test_rolling_shutter_pose_step(gpu_factory, mode):
    """the rolling-shutter pose passes take the corners at their row times: every view keeps its pose, and the poses move off the global
    shutter's towards the truth at the frame time"""
    B, off, ids, uv, vel = rs_scene(RAT, K_CAL, n_views=12, seed=67)
    frame_t = np.arange(12) * 0.05
    res = {}
    for ld in (0.0, LINE_DELAY):
        g = gpu_factory(); g.set_camera(RAT, K_CAL, W, H); g.set_board_points(B); g.set_pose_error(mode)
        g.set_pose_rolling_shutter(ld, frame_t if ld > 0 else None)
        res[ld] = g.estimate_board_poses(off, ids, uv)
        assert res[ld][3].all()
    assert np.isfinite(res[LINE_DELAY][0]).all() and np.abs(res[LINE_DELAY][1] - res[0.0][1]).max() > 0.0


# ---- camera calibration ---------------------------------------------------------------------------------------------------------------
def _rays():
    th = np.radians(np.linspace(0.0, 45.0, 60)); ph = np.linspace(0.0, 2 * np.pi, 60)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


def test_calibration_recovers_the_camera(gpu_factory):
    B, off, ids, uv, q_true, p_true = scene(RAT, K_CAL, n_views=36, seed=3)
    r = _api(gpu_factory, B).calibrate_camera(RAT, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and r["used"].all() and r["intrinsics"].size == 13
    assert np.abs(r["intrinsics"][10:]).max() > 0.0                          # stage 1 frees k4..k6
    px = cm.project(RAT, r["intrinsics"], _rays())[0]
    assert np.abs(px - cm.project(RAT, K_CAL, _rays())[0]).max() < 1e-4       # the same camera over the calibrated field
    assert np.abs(r["intrinsics"][[0, 3, 4]] - K_CAL[[0, 3, 4]]).max() < 1e-4 * K_CAL[0]
    assert _qdiff(r["q_wc"], q_true).max() < 1e-6 and np.abs(r["p_wc"] - p_true).max() < 1e-6 and s["final_reproj_error"] < 1e-5


def test_rolling_shutter_calibration_recovers_the_camera(gpu_factory):
    B, off, ids, uv, vel = rs_scene(RAT, K_CAL, n_views=36, seed=67, noise_px=0.0)
    g = gpu_factory(); g.set_camcal_rolling_shutter(LINE_DELAY, w_u=vel)
    r = _calibrate(g, RAT, dict(board=B, off=off, ids=ids, uv=uv))
    assert r["summary"]["success"] == 1 and r["used"].all()
    assert np.abs(cm.project(RAT, r["intrinsics"], _rays())[0] - cm.project(RAT, K_CAL, _rays())[0]).max() < 1e-4


def test_calibrate_camera_cli_output_feeds_the_hot_cli(tmp_path):
    B, off, ids, uv, q_true, p_true = scene(RAT, K_CAL, n_views=40, seed=17, noise_px=0.1)
    corners = str(tmp_path / "corners.uson")
    _write_corner_file(corners, B, off, ids, uv)
    out = subprocess.run([CAL_CLI, "--input_corners=" + corners, "--camera_model_to_calibrate=PINHOLE_RATIONAL", "--save_path_calib_dataset=" + str(tmp_path / "cam"),
                          "--grid_size=0.001"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr + out.stdout
    assert "PINHOLE_RATIONAL model: Radial distortion 1: " in out.stdout and "Radial distortion 6: " in out.stdout
    cam = json.load(open(str(tmp_path / "cam.json")))
    assert cam["intrinsic_type"] == "PINHOLE_RATIONAL" and cam["final_reproj_error"] < 0.2
    i = cam["intrinsics"]
    got = np.array([i["focal_length"], i["aspect_ratio"], 0.0, i["principal_pt_x"], i["principal_pt_y"]] + [i[f"radial_distortion_{j}"] for j in (1, 2, 3)] +
                   [i["tangential_distortion_1"], i["tangential_distortion_2"]] + [i[f"radial_distortion_{j}"] for j in (4, 5, 6)])
    paths = iof.write_dataset_files(syn.make_dataset(_tiny(K_WIDE, n_frames=8)), str(tmp_path / "seq"))
    paths["camera_calibration_json"] = str(tmp_path / "cam.json")
    out = subprocess.run(_args(paths, str(tmp_path), ["--parse_only"]), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == RAT and np.allclose(s["intrinsics"], got, rtol=1e-12, atol=0)


def test_opencv_import_feeds_the_hot_cli(tmp_path):
    """an OpenCV FileStorage calibration -> opencv_to_json -> the hot CLI (board poses estimated on the GPU, the rotation initialiser, the
    spline solve) on a sequence projected through the imported camera"""
    K = np.array([[K_WIDE[0], 0.0, K_WIDE[3]], [0.0, K_WIDE[0] * K_WIDE[1], K_WIDE[4]], [0.0, 0.0, 1.0]])
    D = [K_WIDE[5], K_WIDE[6], K_WIDE[8], K_WIDE[9], K_WIDE[7], K_WIDE[10], K_WIDE[11], K_WIDE[12]]
    src, cam = tmp_path / "calib.yaml", str(tmp_path / "cam.json")
    src.write_text(_opencv_yaml(K, D, W=960, H=540))
    out = subprocess.run([sys.executable, "-m", "openimucameracalibrator_b200.opencv_to_json", "--input", str(src), "--output", cam, "--fps", "30"],
                         capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    ds = syn.make_dataset(_tiny(K_WIDE, n_frames=30, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
    paths = iof.write_dataset_files(ds, str(tmp_path / "seq"))
    paths["camera_calibration_json"] = cam
    paths.pop("pose_dataset_json", None)
    out = subprocess.run(_args(paths, str(tmp_path), []), capture_output=True, text=True)
    assert out.returncode == 0, out.stderr + out.stdout
    res = json.load(open(str(tmp_path / "result.json")))
    assert res
