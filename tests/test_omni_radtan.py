"""OMNI_RADIAL_TANGENTIAL (Kalibr's omni-radtan) on the CPU: the NumPy model against the oracle, the two exact identities that pin the
formula (zero distortion = EXTENDED_UNIFIED with alpha = xi / (1 + xi), beta = 1, f_eucm = f / (1 + xi); xi = 0 = PINHOLE_RADIAL_TANGENTIAL
with k3 = 0), the product's closed-form Jacobians against central differences and the oracle's autodiff, the product's un-projections,
the CLI's camera reader, and the oracle's spline LM and camera calibration on noise-free data.  The oracle with this model is
tests/omni_radtan/omni_oracle.cpp: the unchanged CPU oracle with the model added beside it (`omni_oracle`, `omni_tangent_oracle`)."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from helpers import F_STAGE1
from test_camera_calibration import TIGHT, H, W, _api, _qdiff, scene
from wide_angle_support import product_bearings

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
DP = ctypes.POINTER(ctypes.c_double)
OMNI = cm.OMNI_RADIAL_TANGENTIAL
# a Kalibr-like omni-radtan calibration of a ~180 degree lens, and one with xi < 1
K17 = np.array([810.0, 1.002, 0.0, 489.5, 272.0, 1.7, -0.2, 0.05, 1e-4, -1.5e-4])
K08 = np.array([684.0, 1.0, 0.0, 479.1, 274.5, 0.8, -0.05, 0.01, 2e-4, -1e-4])
KS = [K17, K08]
KS_IDS = ["xi1.7", "xi0.8"]


def _w(xi):
    return xi if xi <= 1.0 else 1.0 / xi


def _edge_deg(xi):
    """angle off the optical axis of the domain edge z = -w |p|"""
    return np.degrees(np.arccos(-_w(xi)))


def _dirs(th_deg, rng):
    th = np.radians(th_deg); ph = rng.uniform(0, 2 * np.pi, th.size)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


def _points(k, seed):
    """points over the whole sphere at several distances, points behind the camera inside the domain (for xi > 1), and points
    1e-6 rad either side of the domain edge"""
    rng = np.random.default_rng(seed)
    e = _edge_deg(k[5])
    th = np.concatenate([rng.uniform(0, 180, 300), rng.uniform(90, e, 100), np.full(50, e - np.degrees(1e-6)), np.full(50, e + np.degrees(1e-6))])
    return _dirs(th, rng) * rng.uniform(0.2, 5.0, (th.size, 1)), th


_LIBS = {}


def _omni_oracle_lib(tangent=False):
    """the CPU oracle with OMNI_RADIAL_TANGENTIAL (and the rolling-shutter camera calibration; with `tangent`, the tangent reprojection error
    instead), built once per process"""
    if tangent not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_omni_oracle_"), "libomni_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + (["-DOMNI_TANGENT"] if tangent else []) +
                              ["-o", out, os.path.join(HERE, "omni_radtan", "omni_oracle.cpp")])
        _LIBS[tangent] = ctypes.CDLL(out)
    return _LIBS[tangent]


def omni_oracle():
    return capi.CApi(_omni_oracle_lib(), "icco_", 0)


def omni_tangent_oracle():
    return capi.CApi(_omni_oracle_lib(tangent=True), "icco_", 0)


def _oracle_project(model, k, p):
    px = np.zeros(2); kk = np.zeros(10); kk[: len(k)] = k
    ok = _omni_oracle_lib().icco_project(ctypes.c_int(model), kk.ctypes.data_as(DP), np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(DP), px.ctypes.data_as(DP), ctypes.c_int(1))
    return bool(ok), px


@pytest.fixture(scope="module")
def hm(tmp_path_factory):
    """the product's __host__ __device__ camera math compiled for the CPU"""
    out = tmp_path_factory.mktemp("omni_hm") / "libhost_math.so"
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets", "-o", str(out),
                           os.path.join(HERE, "host_math", "host_math.cu")])
    return ctypes.CDLL(str(out))


@pytest.fixture(scope="module")
def oad(tmp_path_factory):
    """the oracle's projection on dual numbers"""
    out = tmp_path_factory.mktemp("omni_oad") / "liboad.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(out), os.path.join(HERE, "omni_radtan", "oracle_autodiff_project.cpp")])
    return ctypes.CDLL(str(out))


def _hm_project(hm, model, k, p):
    out = np.zeros(28); kk = np.zeros(10); kk[: len(k)] = k
    rc = hm.hm_project(ctypes.c_int(model), kk.ctypes.data_as(DP), np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(DP), ctypes.c_int(1), out.ctypes.data_as(DP))
    assert rc & 2, "project() and project_with_k() disagree"
    return bool(rc & 1), out[:2].copy(), out[2:8].reshape(2, 3).copy(), out[8:].reshape(2, 10).copy()


def _oad_project(oad, model, k, p):
    px, Jp, Jk = np.zeros(2), np.zeros(6), np.zeros(20); kk = np.zeros(10); kk[: len(k)] = k
    ok = oad.oad_project(ctypes.c_int(model), kk.ctypes.data_as(DP), np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(DP), px.ctypes.data_as(DP),
                         Jp.ctypes.data_as(DP), Jk.ctypes.data_as(DP))
    return bool(ok), px, Jp.reshape(2, 3), Jk.reshape(2, 10)


def test_model_tables():
    assert cm.MODEL_NAMES[OMNI] == "OMNI_RADIAL_TANGENTIAL" and cm.MODEL_IDS["OMNI_RADIAL_TANGENTIAL"] == 7 and cm.NUM_PARAMS[OMNI] == 10


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_numpy_and_oracle_agree_with_the_same_domain(k):
    pts, th = _points(k, 1)
    uv, valid = cm.project(OMNI, k, pts)
    e = _edge_deg(k[5])
    assert (valid == (th < e)).all()                                      # the domain is a cone about the optical axis
    if k[5] > 1.0:
        assert (valid & (pts[:, 2] < 0)).sum() > 100                      # behind the camera, inside the domain
    for i, p in enumerate(pts):
        ok, px = _oracle_project(OMNI, k, p)
        assert ok == bool(valid[i])
        if ok:
            assert np.abs(px - uv[i]).max() <= 1e-13 * np.abs(uv[i]).max()


def _eucm(k):
    xi = k[5]
    return np.array([k[0] / (1 + xi), k[1], k[2] / (1 + xi), k[3], k[4], xi / (1 + xi), 1.0])


@pytest.mark.parametrize("xi", [0.3, 0.8, 1.0, 1.7, 2.5])
def test_zero_distortion_is_the_extended_unified_model(hm, xi):
    k = np.array([700.0, 1.01, 0.4, 480.0, 270.0, xi, 0.0, 0.0, 0.0, 0.0])
    pts, th = _points(k, int(10 * xi))
    e = _edge_deg(xi)
    for p, t in zip(pts, th):
        for project in (_oracle_project, lambda m, kk, pp: _hm_project(hm, m, kk, pp)[:2]):
            ok, px = project(OMNI, k, p)
            ok_e, px_e = project(cm.EXTENDED_UNIFIED, _eucm(k), p)
            assert ok == ok_e
            if ok and t < e - 1e-3:     # (1e-6 rad from the edge of xi <= 1, z + xi |p| cancels to 1e-6 |p|: the two statements round apart)
                assert np.abs(px - px_e).max() <= 1e-12 * np.abs(px_e).max()


def test_xi_zero_is_the_pinhole_radial_tangential_model(hm):
    k = np.array([440.0, 1.01, 0.2, 480.0, 270.0, 0.0, -0.1, 0.02, 1e-3, -2e-3])
    kp = np.array([440.0, 1.01, 0.2, 480.0, 270.0, -0.1, 0.02, 0.0, 1e-3, -2e-3])
    rng = np.random.default_rng(3)
    pts = _dirs(rng.uniform(0, 60, 300), rng) * rng.uniform(0.2, 5.0, (300, 1))
    for p in pts:
        ok, px = _oracle_project(OMNI, k, p)
        ok_p, px_p = _oracle_project(cm.PINHOLE_RADIAL_TANGENTIAL, kp, p)
        assert ok and ok_p and np.abs(px - px_p).max() <= 1e-13 * np.abs(px_p).max()
        ok, px, J, Jk = _hm_project(hm, OMNI, k, p)
        ok_p, px_p, J_p, Jk_p = _hm_project(hm, cm.PINHOLE_RADIAL_TANGENTIAL, kp, p)
        assert ok and ok_p and np.abs(px - px_p).max() <= 1e-13 * np.abs(px_p).max()
        assert np.abs(J - J_p).max() <= 1e-12 * np.abs(J_p).max()
        # shared columns: f, ar, skew, cx, cy, k1, k2, t1, t2
        assert np.abs(Jk[:, [0, 1, 2, 3, 4, 6, 7, 8, 9]] - Jk_p[:, [0, 1, 2, 3, 4, 5, 6, 8, 9]]).max() <= 1e-12 * np.abs(Jk_p).max()


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_device_jacobians_match_central_differences_and_autodiff(hm, oad, k):
    assert hm.hm_num_params(OMNI) == 10
    rng = np.random.default_rng(5)
    e = _edge_deg(k[5])
    hi = e - 3.0 if k[5] > 1.0 else 100.0            # xi < 1: pixels grow without bound towards the edge
    pts = _dirs(rng.uniform(0, hi, 200), rng) * rng.uniform(0.3, 3.0, (200, 1))
    uv_np, valid = cm.project(OMNI, k, pts)
    assert valid.all()
    for p, uv_ref in zip(pts, uv_np):
        ok, uv, J, Jk = _hm_project(hm, OMNI, k, p)
        ok_a, uv_a, J_a, Jk_a = _oad_project(oad, OMNI, k, p)
        assert ok and ok_a
        assert np.abs(uv - uv_ref).max() <= 1e-13 * np.abs(uv_ref).max() and np.abs(uv_a - uv_ref).max() <= 1e-13 * np.abs(uv_ref).max()
        assert np.abs(J - J_a).max() <= 1e-11 * np.abs(J_a).max()
        assert np.abs(Jk - Jk_a).max() <= 1e-11 * np.abs(Jk_a).max()
        Jfd = np.zeros((2, 3))
        for d in range(3):
            h = 1e-6 * max(1.0, abs(p[d])); dp = np.zeros(3); dp[d] = h
            Jfd[:, d] = (cm.project(OMNI, k, (p + dp)[None])[0][0] - cm.project(OMNI, k, (p - dp)[None])[0][0]) / (2 * h)
        assert np.abs(J - Jfd).max() < 2e-6 * max(1.0, np.abs(Jfd).max())
        for q in range(10):
            h = 1e-6 * max(1.0, abs(k[q])); kp, km = k.copy(), k.copy(); kp[q] += h; km[q] -= h
            fd = (cm.project(OMNI, kp, p[None])[0][0] - cm.project(OMNI, km, p[None])[0][0]) / (2 * h)
            assert np.abs(Jk[:, q] - fd).max() < 2e-6 * max(1.0, np.abs(fd).max()), q


def test_points_outside_the_domain_fail_in_the_device_math(hm):
    for k in KS:
        pts, th = _points(k, 7)
        for p, t in zip(pts, th):
            ok, _, J, _ = _hm_project(hm, OMNI, k, p)
            assert ok == (t < _edge_deg(k[5]))
            if not ok:
                assert not J.any()


@pytest.mark.parametrize("k", [K17, np.r_[K08[:6], 0.0, 0.0, 0.0, 0.0], np.r_[K17[:5], 1.0, 0.0, 0.0, 0.0, 0.0], np.r_[K17[:5], 2.0, 0.0, 0.0, 0.0, 0.0]],
                         ids=["xi1.7", "xi0.8_undistorted", "xi1_undistorted", "xi2_undistorted"])
def test_bearings_round_trip_up_to_the_domain_edge(k):
    e = _edge_deg(k[5])
    rng = np.random.default_rng(11)
    th = np.concatenate([rng.uniform(0, e - 1.0, 400), np.full(20, e - 1.0)])
    rays = _dirs(th, rng)
    px, valid = cm.project(OMNI, k, rays)
    assert valid.all() and (th > 90.0).sum() > 100
    b, ok = product_bearings(OMNI, k, px)
    assert ok.all()
    assert np.abs(b - rays).max() < 1e-8
    assert np.abs(cm.project(OMNI, k, b)[0] - px).max() < 1e-6


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_unproject_gn_round_trips_rays_in_front(hm, k):
    rng = np.random.default_rng(13)
    rays = _dirs(rng.uniform(0, 75, 300), rng)
    px, valid = cm.project(OMNI, k, rays)
    assert valid.all()
    kk = np.ascontiguousarray(k)
    for r, (u, v) in zip(rays, px):
        xy = np.zeros(2)
        assert hm.hm_unproject(ctypes.c_int(OMNI), kk.ctypes.data_as(DP), ctypes.c_double(u), ctypes.c_double(v), xy.ctypes.data_as(DP)) == 1
        assert np.abs(xy - r[:2] / r[2]).max() < 1e-9 * max(1.0, np.abs(r[:2] / r[2]).max())


def _tiny(k=K17, **kw):
    return syn.tiny_config(OMNI, tuple(k), **kw)


def test_cli_reads_the_written_camera(tmp_path):
    ds = syn.make_dataset(_tiny(n_frames=8))
    paths = iof.write_dataset_files(ds, str(tmp_path))
    cam = json.load(open(paths["camera_calibration_json"]))
    assert cam["intrinsic_type"] == "OMNI_RADIAL_TANGENTIAL" and cam["intrinsics"]["xi"] == K17[5]
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/result.json", f"--output_path={tmp_path}", "--parse_only"]
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == 7
    k_expected = K17.copy(); k_expected[2] = 0.0                          # `skew` is written, never read
    assert np.array_equal(np.array(s["intrinsics"]), k_expected)
    del cam["intrinsics"]["xi"]
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode != 0 and "missing key 'xi'" in out.stderr


def test_oracle_spline_lm_recovers_the_truth():
    ds = syn.make_dataset(_tiny(n_frames=40, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
    o = omni_oracle(); capi.load_dataset(o, ds)
    qt = ds["truth"]["T_i_c"]
    rot_err = lambda q: np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))   # noqa: E731
    assert rot_err(o.get_T_i_c()) > 0.5
    s = o.optimize(50, F_STAGE1)
    T = o.get_T_i_c()
    # noise-free corners, but a trajectory that no quintic B-spline holds exactly
    assert rot_err(T) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-5
    assert s.mean_reproj_error < 1e-3


def _centred(k):
    """what stage 1 of the calibration (focal length, xi, k1, k2 free; aspect ratio 1, principal point at the image centre) can solve exactly"""
    k = k.copy(); k[1] = 1.0; k[3], k[4] = W / 2, H / 2; k[8] = k[9] = 0.0
    return k


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_oracle_camera_calibration_recovers_the_intrinsics(k):
    k = _centred(k)
    B, off, ids, uv, q_true, p_true = scene(OMNI, k, seed=3)
    r = _api(omni_oracle, B).calibrate_camera(OMNI, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and s["n_views_used"] == 30 and r["used"].all()
    assert np.abs(r["intrinsics"] - k).max() < 1e-6 * np.abs(k).max()
    assert _qdiff(r["q_wc"], q_true).max() < 1e-8 and np.abs(r["p_wc"] - p_true).max() < 1e-8
    assert s["final_reproj_error"] < 1e-8


def test_omni_oracle_is_the_oracle_for_every_other_model(oracle_factory):
    """the substitutions of omni_oracle.cpp leave the oracle's own models untouched: bit-identical evaluations and camera calibrations"""
    ds = syn.make_dataset(syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), n_frames=12))
    a, b = oracle_factory(), omni_oracle()
    capi.load_dataset(a, ds); capi.load_dataset(b, ds)
    for x, y in zip(a.evaluate(F_STAGE1, hessian=True), b.evaluate(F_STAGE1, hessian=True)):
        assert np.array_equal(x, y)
    k = np.array([437.1, 1.0, 0.0, W / 2, H / 2, -0.05, 0.01, -0.003, 1e-3, -2e-3])
    B, off, ids, uv, _, _ = scene(cm.PINHOLE_RADIAL_TANGENTIAL, k, seed=4, noise_px=0.2)
    ra = _api(oracle_factory, B).calibrate_camera(cm.PINHOLE_RADIAL_TANGENTIAL, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    rb = _api(omni_oracle, B).calibrate_camera(cm.PINHOLE_RADIAL_TANGENTIAL, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    for key in ("intrinsics", "q_wc", "p_wc", "view_error_px"):
        assert np.array_equal(ra[key], rb[key]), key
