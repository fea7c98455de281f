"""SCARAMUZZA (Scaramuzza's omnidirectional polynomial model as OCamCalib calibrates it) on the CPU: the NumPy model against the oracle and
np.roots, the two exact identities that pin the statement (a constant polynomial with d = 0 = PINHOLE [a0, c, a0 e, cx, cy]; a2 = -1/(4 a0)
= the stereographic projection = OMNI_RADIAL_TANGENTIAL with xi = 1, f = 2 a0), the product's implicit-function Jacobians against the
oracle's autodiff and central differences, the closed-form bearings, the oracle's camera calibration and spline LM, the OCamCalib importer
and the CLI's camera reader.  The oracle with this model is tests/scaramuzza/scaramuzza_oracle.cpp: the unchanged CPU oracle with the model
added beside it (`scara_oracle`, `scara_tangent_oracle`)."""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import ocamcalib_to_json as o2j
from openimucameracalibrator_b200 import synthetic as syn
from helpers import F_STAGE1
from test_camera_calibration import TIGHT, H, W, _api, _qdiff, scene
from test_omni_radtan import _oracle_project as _omni_oracle_project
from wide_angle_support import product_bearings

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
DP = ctypes.POINTER(ctypes.c_double)
SCARA = cm.SCARAMUZZA
# [a0, c, e, cx, cy, a2, a3, a4, d]
K_NEAR = np.array([450.0, 1.001, 2e-4, 480.0, 270.0, -1e-5, 0.0, 0.0, 0.0])                  # near-pinhole; rho_max = inf
K_FISH = np.array([250.0, 0.998, -3e-4, 480.0, 270.0, -1.1e-3, 2e-7, -5e-10, 1e-4])         # 200 degrees across the diagonal; rho_max = inf, a4 < 0
K_FIN = np.array([300.0, 1.002, 1e-4, 480.0, 270.0, -8e-4, 1e-7, 2e-9, -2e-4])              # rho_max = 537 px: a cone of 65 degrees
K_A3 = np.array([280.0, 1.0, 0.0, 480.0, 270.0, -9e-4, 5e-7, 0.0, 0.0])                     # a4 = 0, rho_max = 1122 px: a cone of 97 degrees
KS = [K_NEAR, K_FISH, K_FIN, K_A3]
KS_IDS = ["near_pinhole", "fisheye", "finite_rho_max", "cubic"]


def _edge_deg(k):
    """angle off the optical axis of the domain edge (180 for rho_max = inf and a non-constant polynomial)"""
    rm = cm.scaramuzza_rho_max(k)
    if np.isfinite(rm):
        return np.degrees(np.arctan2(rm, cm.scaramuzza_F(k, rm)))
    return 90.0 if not k[5:8].any() else 180.0


def _dirs(th_deg, rng):
    th = np.radians(th_deg); ph = rng.uniform(0, 2 * np.pi, th.size)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


def _points(k, seed, n=400):
    """points over the whole sphere at several distances (behind the camera and past 90 degrees included), at least 1e-3 rad from the
    domain edge, plus points on the optical axis (r = 0 exactly) in front and behind, and at r = 1e-300 in front"""
    rng = np.random.default_rng(seed)
    e = _edge_deg(k)
    th = rng.uniform(0, 179.9, n)
    th = th[np.abs(th - e) > np.degrees(1e-3)]
    pts = _dirs(th, rng) * rng.uniform(0.2, 5.0, (th.size, 1))
    axis = np.array([[0.0, 0.0, 1.3], [0.0, 0.0, -0.7], [1e-300, 0.0, 2.0], [0.0, -1e-300, 0.4]])
    return np.concatenate([pts, axis])


_LIBS = {}


def _scara_oracle_lib(tangent=False):
    """the CPU oracle with SCARAMUZZA (and the rolling-shutter camera calibration; with `tangent`, the tangent reprojection error instead),
    built once per process"""
    if tangent not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_scara_oracle_"), "libscara_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread"] + (["-DSCARAMUZZA_TANGENT"] if tangent else []) +
                              ["-o", out, os.path.join(HERE, "scaramuzza", "scaramuzza_oracle.cpp")])
        _LIBS[tangent] = ctypes.CDLL(out)
    return _LIBS[tangent]


def scara_oracle():
    return capi.CApi(_scara_oracle_lib(), "icco_", 0)


def scara_tangent_oracle():
    return capi.CApi(_scara_oracle_lib(tangent=True), "icco_", 0)


def _oracle_project(model, k, p):
    px = np.zeros(2); kk = np.zeros(10); kk[: len(k)] = k
    ok = _scara_oracle_lib().icco_project(ctypes.c_int(model), kk.ctypes.data_as(DP), np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(DP), px.ctypes.data_as(DP), ctypes.c_int(1))
    return bool(ok), px


@pytest.fixture(scope="module")
def hm(tmp_path_factory):
    """the product's __host__ __device__ camera math compiled for the CPU"""
    out = tmp_path_factory.mktemp("scara_hm") / "libhost_math.so"
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets", "-o", str(out),
                           os.path.join(HERE, "host_math", "host_math.cu")])
    return ctypes.CDLL(str(out))


@pytest.fixture(scope="module")
def oad(tmp_path_factory):
    """the oracle's projection on dual numbers"""
    out = tmp_path_factory.mktemp("scara_oad") / "liboad.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(out), os.path.join(HERE, "scaramuzza", "oracle_autodiff_project.cpp")])
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
    assert cm.MODEL_NAMES[SCARA] == "SCARAMUZZA" and cm.MODEL_IDS["SCARAMUZZA"] == 8 and cm.NUM_PARAMS[SCARA] == 9


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_numpy_and_oracle_agree_with_the_same_domain(k):
    pts = _points(k, 1)
    uv, valid = cm.project(SCARA, k, pts)
    th = np.degrees(np.arctan2(np.hypot(pts[:, 0], pts[:, 1]), pts[:, 2]))
    assert (valid == (th < _edge_deg(k))).all()                               # the domain is a cone about the optical axis
    assert valid[-4:].tolist() == [True, False, True, True]                   # on the axis: z > 0
    if _edge_deg(k) > 90.0:
        assert (valid & (pts[:, 2] < 0)).sum() > 5                            # behind the camera, inside the domain
    for i, p in enumerate(pts):
        ok, px = _oracle_project(SCARA, k, p)
        assert ok == bool(valid[i])
        if ok:
            assert np.abs(px - uv[i]).max() <= 1e-13 * np.abs(uv[i]).max()


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_numpy_rho_max_and_root_agree_with_np_roots(k):
    rm = cm.scaramuzza_rho_max(k)
    a0, a2, a3, a4 = k[0], k[5], k[6], k[7]
    F = lambda rho: a0 + a2 * rho ** 2 + a3 * rho ** 3 + a4 * rho ** 4        # noqa: E731
    dense = np.linspace(1e-3, 5000.0, 200001)                                 # F(rho) / rho first stops falling at rho_max
    slope = np.diff(F(dense) / dense)
    assert (np.isfinite(rm) and abs(dense[np.argmax(slope >= 0)] - rm) < 0.05) or (not np.isfinite(rm) and (slope < 0).all())
    pts = _points(k, 2, 200)
    r, z = np.hypot(pts[:, 0], pts[:, 1]), pts[:, 2]
    s, valid = cm.scaramuzza_scale(k, r, z)
    for si, ri, zi, vi in zip(s, r, z, valid):
        if not vi or ri == 0.0 or ri < 1e-200:
            continue
        roots = np.roots([a4 * ri ** 4, a3 * ri ** 3, a2 * ri ** 2, -zi, a0])
        real = roots.real[(np.abs(roots.imag) <= 1e-9 * np.abs(roots)) & (roots.real > 0) & (roots.real * ri < rm)]
        assert real.size == 1                                                 # exactly one root on the branch
        assert abs(real[0] - si) <= 1e-9 * si
    on_axis = (r < 1e-200) & valid
    assert np.abs(s[on_axis] - a0 / z[on_axis]).max() <= 4e-16 * np.abs(s[on_axis]).max()   # s = a0 / z on the principal ray


def _pinhole_of(k):
    return np.array([k[0], k[1], k[0] * k[2], k[3], k[4], 0.0, 0.0])


@pytest.mark.parametrize("seed", [0, 1])
def test_constant_polynomial_is_the_pinhole_model(hm, seed):
    rng = np.random.default_rng(seed)
    k = np.array([rng.uniform(200, 900), rng.uniform(0.98, 1.02), rng.uniform(-1e-3, 1e-3), 480.0, 270.0, 0.0, 0.0, 0.0, 0.0])
    pts = np.concatenate([_dirs(rng.uniform(0, 180, 400), rng) * rng.uniform(0.2, 5.0, (400, 1)), [[0, 0, 1.0], [0, 0, -1.0], [1e-300, 0, 1.0]]])
    pts = pts[np.abs(pts[:, 2]) > 1e-3 * np.linalg.norm(pts, axis=1)]
    uv, valid = cm.project(SCARA, k, pts)
    assert (valid == (pts[:, 2] > 0)).all()                                   # the domain z > 0
    uv_p, _ = cm.project(cm.PINHOLE, _pinhole_of(k), pts)
    assert np.abs(uv - uv_p)[valid].max() <= 1e-12 * np.abs(uv_p[valid]).max()
    for p, v in zip(pts, valid):
        for project in (_oracle_project, lambda m, kk, pp: _hm_project(hm, m, kk, pp)[:2]):
            ok, px = project(SCARA, k, p)
            ok_p, px_p = project(cm.PINHOLE, _pinhole_of(k), p)
            assert ok == bool(v) and ok_p
            if ok:
                assert np.abs(px - px_p).max() <= 1e-12 * np.abs(px_p).max()


@pytest.mark.parametrize("a0", [150.0, 320.0, 700.0])
def test_stereographic_polynomial_is_the_omni_model_at_xi_one(hm, a0):
    k = np.array([a0, 1.0, 0.0, 480.0, 270.0, -0.25 / a0, 0.0, 0.0, 0.0])
    ko = np.array([2 * a0, 1.0, 0.0, 480.0, 270.0, 1.0, 0.0, 0.0, 0.0, 0.0])
    rng = np.random.default_rng(int(a0))
    th = np.concatenate([rng.uniform(0, 179.0, 400), rng.uniform(90.0, 179.0, 200)])      # past 90 and past 180 degrees of field
    pts = np.concatenate([_dirs(th, rng) * rng.uniform(0.2, 5.0, (th.size, 1)), [[0, 0, 1.0], [0, 0, -1.0], [1e-300, 0, 2.0]]])
    uv, valid = cm.project(SCARA, k, pts)
    uv_o, valid_o = cm.project(cm.OMNI_RADIAL_TANGENTIAL, ko, pts)
    assert np.array_equal(valid, valid_o) and valid[:-2].all() and not valid[-2]          # every point except the negative axis
    assert np.abs(uv - uv_o)[valid].max() <= 1e-12 * np.abs(uv_o[valid]).max()
    hm_project = lambda m, kk, pp: _hm_project(hm, m, kk, pp)[:2]             # noqa: E731
    for p, v in zip(pts, valid):
        for project, project_o in ((_oracle_project, _omni_oracle_project), (hm_project, hm_project)):
            ok, px = project(SCARA, k, p)
            ok_o, px_o = project_o(cm.OMNI_RADIAL_TANGENTIAL, ko, p)
            assert ok == ok_o == bool(v)
            if ok:
                assert np.abs(px - px_o).max() <= 1e-12 * np.abs(px_o).max()


def _fd5(f, x, h):
    """five-point central difference"""
    return (-f(x + 2 * h) + 8 * f(x + h) - 8 * f(x - h) + f(x - 2 * h)) / (12 * h)


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_device_jacobians_match_autodiff_and_central_differences(hm, oad, k):
    assert hm.hm_num_params(SCARA) == 9
    pts = _points(k, 5, 150)
    uv_np, valid = cm.project(SCARA, k, pts)
    # away from the domain edge, and no further out than a few image radii
    keep = valid & (np.abs(uv_np - k[3:5]).max(1) < 1500.0)
    if np.isfinite(cm.scaramuzza_rho_max(k)):
        s, _ = cm.scaramuzza_scale(k, np.hypot(pts[:, 0], pts[:, 1]), pts[:, 2])
        keep &= s * np.hypot(pts[:, 0], pts[:, 1]) < 0.98 * cm.scaramuzza_rho_max(k)
    assert keep.sum() > 40 and (keep & (pts[:, 0] == 0) & (pts[:, 1] == 0)).any()
    for p, uv_ref in zip(pts[keep], uv_np[keep]):
        ok, uv, J, Jk = _hm_project(hm, SCARA, k, p)
        ok_a, uv_a, J_a, Jk_a = _oad_project(oad, SCARA, k, p)
        assert ok and ok_a
        assert np.abs(uv - uv_ref).max() <= 1e-13 * np.abs(uv_ref).max() and np.abs(uv_a - uv_ref).max() <= 1e-13 * np.abs(uv_ref).max()
        assert np.abs(J - J_a).max() <= 1e-9 * np.abs(J_a).max()
        for q in range(9):
            assert np.abs(Jk[:, q] - Jk_a[:, q]).max() <= 1e-9 * max(np.abs(Jk_a[:, q]).max(), 1e-300), q
        assert not Jk[:, 9].any() and not Jk_a[:, 9].any()
        h = 1e-4 * max(1.0, np.linalg.norm(p))
        for d in range(3):
            e = np.zeros(3); e[d] = 1.0
            fd = _fd5(lambda t: cm.project(SCARA, k, (p + t * e)[None])[0][0], 0.0, h)
            assert np.abs(J[:, d] - fd).max() <= 1e-9 * max(1.0, np.abs(J).max()), d
        rho = max(np.hypot(*(uv_ref - k[3:5])), 1.0)
        for q in range(9):
            e = np.zeros(9); e[q] = 1.0
            hq = 1e-4 * k[0] / rho ** max(q - 3, 0) if q in (0, 5, 6, 7) else 1e-3 * max(abs(k[q]), 1.0)   # a_i moves F(rho) by 1e-4 a0
            fd = _fd5(lambda t: cm.project(SCARA, k + t * e, p[None])[0][0], 0.0, hq)
            assert np.abs(Jk[:, q] - fd).max() <= 1e-9 * max(np.abs(fd).max(), 1e-3 / hq), q     # (or 1e-12 px over the step)


def test_points_outside_the_domain_fail_in_the_device_math(hm):
    for k in KS:
        pts = _points(k, 7, 200)
        _, valid = cm.project(SCARA, k, pts)
        assert (~valid).any()
        for p, v in zip(pts, valid):
            ok, _, J, Jk = _hm_project(hm, SCARA, k, p)
            assert ok == bool(v)
            if not ok:
                assert not J.any() and not Jk.any()


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_bearings_round_trip(k):
    rng = np.random.default_rng(11)
    e = _edge_deg(k)
    th = rng.uniform(0, min(e, 179.0) - 0.5, 600)
    rays = _dirs(th, rng)
    px, valid = cm.project(SCARA, k, rays)
    assert valid.all()
    b, ok = product_bearings(SCARA, k, px)
    assert ok.all()
    assert np.abs(b - rays).max() < 1e-12                                     # unproject_bearing(project(p)) = p / |p|
    # project(unproject_bearing(px)) = px over the whole image, past 90 degrees included where the lens sees that far
    u, v = np.meshgrid(np.linspace(0, W, 49), np.linspace(0, H, 28))
    grid = np.stack([u.ravel(), v.ravel()], -1)
    b, ok = product_bearings(SCARA, k, grid)
    det = k[1] - k[8] * k[2]
    sensor = np.stack([(k[1] * (grid[:, 0] - k[3]) - k[2] * (grid[:, 1] - k[4])) / det, ((grid[:, 1] - k[4]) - k[8] * (grid[:, 0] - k[3])) / det], -1)
    inside = np.linalg.norm(sensor, axis=1) < cm.scaramuzza_rho_max(k)
    assert np.array_equal(ok.astype(bool), inside)                            # pixels beyond rho_max are refused
    px2, valid2 = cm.project(SCARA, k, b[inside])
    assert valid2.all() and np.abs(px2 - grid[inside]).max() < 1e-9
    if k is K_FISH:
        assert (b[inside][:, 2] < 0).sum() > 50                               # past 90 degrees
    if k is K_FIN:
        assert (~inside).sum() > 0


def test_bearings_refuse_a_singular_stretch():
    k = K_FISH.copy(); k[1] = 0.5; k[2] = 2.0; k[8] = 0.25                    # det A = c - d e = 0
    _, ok = product_bearings(SCARA, k, np.array([[500.0, 300.0], [480.0, 270.0]]))
    assert not ok.any()


def test_scara_oracle_is_the_oracle_for_every_other_model(oracle_factory):
    """the substitutions of scaramuzza_oracle.cpp leave the oracle's own models untouched: bit-identical evaluations and camera calibrations"""
    ds = syn.make_dataset(syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), n_frames=12))
    a, b = oracle_factory(), scara_oracle()
    capi.load_dataset(a, ds); capi.load_dataset(b, ds)
    for x, y in zip(a.evaluate(F_STAGE1, hessian=True), b.evaluate(F_STAGE1, hessian=True)):
        assert np.array_equal(x, y)
    k = np.array([437.1, 1.0, 0.0, W / 2, H / 2, -0.05, 0.01, -0.003, 1e-3, -2e-3])
    B, off, ids, uv, _, _ = scene(cm.PINHOLE_RADIAL_TANGENTIAL, k, seed=4, noise_px=0.2)
    ra = _api(oracle_factory, B).calibrate_camera(cm.PINHOLE_RADIAL_TANGENTIAL, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    rb = _api(scara_oracle, B).calibrate_camera(cm.PINHOLE_RADIAL_TANGENTIAL, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    for key in ("intrinsics", "q_wc", "p_wc", "view_error_px"):
        assert np.array_equal(ra[key], rb[key]), key


def _centred(k):
    """what stage 1 of the calibration (a0, a2, a3, a4 free; c = 1, no stretch, principal point at the image centre) can solve exactly"""
    k = k.copy(); k[1] = 1.0; k[2] = k[8] = 0.0; k[3], k[4] = W / 2, H / 2
    return k


@pytest.mark.parametrize("k", [K_NEAR, K_FISH], ids=["near_pinhole", "fisheye"])
def test_oracle_camera_calibration_recovers_the_intrinsics(k):
    k = _centred(k)
    B, off, ids, uv, q_true, p_true = scene(SCARA, k, seed=3)
    r = _api(scara_oracle, B).calibrate_camera(SCARA, W, H, off, ids, uv, grid_size=0.0, **TIGHT)
    s = r["summary"]
    assert s["success"] == 1 and s["n_views_used"] == 30 and r["used"].all()
    px, _ = cm.project(SCARA, r["intrinsics"], _dirs(np.linspace(0, 60, 50), np.random.default_rng(0)))
    px_t, _ = cm.project(SCARA, k, _dirs(np.linspace(0, 60, 50), np.random.default_rng(0)))
    assert np.abs(px - px_t).max() < 1e-6                                     # the same camera
    assert np.abs(r["intrinsics"][:5] - k[:5]).max() < 1e-6 * k[0]
    assert _qdiff(r["q_wc"], q_true).max() < 1e-8 and np.abs(r["p_wc"] - p_true).max() < 1e-8
    assert s["final_reproj_error"] < 1e-8


def _tiny(k=K_FISH, **kw):
    return syn.tiny_config(SCARA, tuple(k), **kw)


def test_oracle_spline_lm_recovers_the_truth():
    ds = syn.make_dataset(_tiny(n_frames=40, corner_noise_px=0.0, imu_noise=False, pose_noise_m=0.0, pose_noise_rad=0.0))
    o = scara_oracle(); capi.load_dataset(o, ds)
    qt = ds["truth"]["T_i_c"]
    rot_err = lambda q: np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))   # noqa: E731
    assert rot_err(o.get_T_i_c()) > 0.5
    s = o.optimize(50, F_STAGE1)
    T = o.get_T_i_c()
    assert rot_err(T) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-5
    assert s.mean_reproj_error < 1e-3


# ---- OCamCalib cameras ------------------------------------------------------------------------------------------------------------------
# an OCamCalib-like calibration of a 1024 x 768 fisheye: pol (ss), invpol, centre (row, column), c d e, height width
OCAM = dict(pol=[-2.44e2, 0.0, 1.3e-3, -1.1e-6, 2.6e-9], invpol=[363.5, 226.2, -3.1, 32.3, 21.1, -3.1, 10.2], row=383.52, col=511.23,
            c=1.000302, d=0.000147, e=-0.000095, height=768, width=1024)


def write_calib_results(path, pol=OCAM["pol"], invpol=OCAM["invpol"]):
    """calib_results.txt in the layout OCamCalib writes"""
    g = lambda v: " ".join(f"{x:.6e}" for x in v)                             # noqa: E731
    with open(path, "w") as f:
        f.write("#polynomial coefficients for the DIRECT mapping function (ocam_model.ss in MATLAB). These are used by cam2world\n\n")
        f.write(f"{len(pol)} {g(pol)} \n\n")
        f.write("#polynomial coefficients for the inverse mapping function (ocam_model.invpol in MATLAB). These are used by world2cam\n\n")
        f.write(f"{len(invpol)} {' '.join(f'{x:.6f}' for x in invpol)} \n\n")
        f.write('#center: "row" and "column", starting from 0 (C convention)\n\n')
        f.write(f"{OCAM['row']:.6f} {OCAM['col']:.6f}\n\n")
        f.write('#affine parameters "c", "d", "e"\n\n')
        f.write(f"{OCAM['c']:.6f} {OCAM['d']:.6f} {OCAM['e']:.6f}\n\n")
        f.write('#image size: "height" and "width"\n\n')
        f.write(f"{OCAM['height']} {OCAM['width']}\n\n")


def _ocam_cam2world(pol, m):
    """OCamCalib's cam2world: pixels (row, column) -> unit vectors in its camera frame"""
    c, d, e = OCAM["c"], OCAM["d"], OCAM["e"]
    invdet = 1.0 / (c - d * e)
    xp = invdet * ((m[:, 0] - OCAM["row"]) - d * (m[:, 1] - OCAM["col"]))
    yp = invdet * (-e * (m[:, 0] - OCAM["row"]) + c * (m[:, 1] - OCAM["col"]))
    r = np.hypot(xp, yp)
    zp = sum(pol[i] * r ** i for i in range(len(pol)))
    v = np.stack([xp, yp, zp], -1)
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _ocam_world2cam_exact(pol, P):
    """OCamCalib's world2cam with the exact root of pol(t |(x, y)|) = t z (OCamCalib's frame) in place of invpol -> (row, column)"""
    out = np.zeros((len(P), 2))
    for i, (x, y, z) in enumerate(P):
        n = np.hypot(x, y)
        coef = [pol[j] * n ** j for j in range(len(pol))]; coef[1] -= z     # pol(t n) - t z
        t = np.roots(coef[::-1])
        t = t.real[(np.abs(t.imag) < 1e-9 * np.abs(t)) & (t.real > 0)].min()
        xp, yp = t * x, t * y
        out[i] = [xp * OCAM["c"] + yp * OCAM["d"] + OCAM["row"], xp * OCAM["e"] + yp + OCAM["col"]]
    return out


def test_ocamcalib_import_projects_as_ocamcalib(tmp_path):
    src, dst = str(tmp_path / "calib_results.txt"), str(tmp_path / "cam.json")
    write_calib_results(src)
    doc = o2j.main(["--input", src, "--output", dst, "--fps", "29.97"])
    cam = json.load(open(dst))
    assert cam == json.loads(json.dumps(doc)) and cam["intrinsic_type"] == "SCARAMUZZA" and cam["fps"] == 29.97
    assert (cam["image_width"], cam["image_height"]) == (1024, 768)
    i = cam["intrinsics"]
    k = np.array([i["focal_length"], i["aspect_ratio"], i["stretch_e"], i["principal_pt_x"], i["principal_pt_y"], i["polynomial_a2"], i["polynomial_a3"],
                  i["polynomial_a4"], i["stretch_d"]])
    pol = OCAM["pol"]
    assert np.array_equal(k, [-pol[0], OCAM["c"], OCAM["e"], OCAM["col"], OCAM["row"], -pol[2], -pol[3], -pol[4], OCAM["d"]])
    rng = np.random.default_rng(2)
    P = _dirs(rng.uniform(0, 95, 300), rng) * rng.uniform(0.3, 4.0, (300, 1))      # this project's frame: x right, y down, z forward
    uv, valid = cm.project(SCARA, k, P)
    assert valid.all()
    P_o = np.stack([P[:, 1], P[:, 0], -P[:, 2]], -1)                          # OCamCalib's frame: (row, column, away from the scene)
    rc = _ocam_world2cam_exact(pol, P_o)
    assert np.abs(uv - rc[:, ::-1]).max() < 1e-9
    # cam2world of those pixels gives the points' directions back, in either frame
    back = _ocam_cam2world(pol, rc)
    assert np.abs(back - P_o / np.linalg.norm(P_o, axis=1, keepdims=True)).max() < 1e-12
    b, ok = product_bearings(SCARA, k, uv)
    assert ok.all() and np.abs(b - np.stack([back[:, 1], back[:, 0], -back[:, 2]], -1)).max() < 1e-12


@pytest.mark.parametrize("pol,msg", [([-2.44e2, 1e-3, 1.3e-3, -1.1e-6, 2.6e-9], "pol[1] != 0"),
                                     ([-2.44e2, 0.0, 1.3e-3, -1.1e-6, 2.6e-9, 1e-13], "degree 5")])
def test_ocamcalib_import_refuses_what_the_model_cannot_hold(tmp_path, pol, msg):
    src = str(tmp_path / "calib_results.txt")
    write_calib_results(src, pol=pol)
    out = subprocess.run([sys.executable, "-m", "openimucameracalibrator_b200.ocamcalib_to_json", "--input", src, "--output", str(tmp_path / "cam.json"), "--fps", "30"],
                         capture_output=True, text=True, cwd=ROOT)
    assert out.returncode != 0 and msg in out.stderr and not os.path.exists(str(tmp_path / "cam.json"))


def _parse_only(paths, tmp_path):
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/result.json", f"--output_path={tmp_path}", "--parse_only"]
    return subprocess.run(args, capture_output=True, text=True)


def test_cli_reads_the_written_camera(tmp_path):
    ds = syn.make_dataset(_tiny(n_frames=8))
    paths = iof.write_dataset_files(ds, str(tmp_path))
    cam = json.load(open(paths["camera_calibration_json"]))
    assert cam["intrinsic_type"] == "SCARAMUZZA" and cam["intrinsics"]["polynomial_a4"] == K_FISH[7] and cam["intrinsics"]["stretch_d"] == K_FISH[8]
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == 8 and np.array_equal(np.array(s["intrinsics"]), K_FISH)
    del cam["intrinsics"]["polynomial_a3"]
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode != 0 and "missing key 'polynomial_a3'" in out.stderr


def test_cli_reads_the_imported_ocamcalib_camera(tmp_path):
    src = str(tmp_path / "calib_results.txt")
    write_calib_results(src)
    paths = iof.write_dataset_files(syn.make_dataset(_tiny(n_frames=8)), str(tmp_path / "seq"))
    paths["camera_calibration_json"] = str(tmp_path / "cam.json")
    doc = o2j.main(["--input", src, "--output", paths["camera_calibration_json"], "--fps", "30"])
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    i = doc["intrinsics"]
    assert s["camera_model"] == 8 and s["intrinsics"] == [i["focal_length"], i["aspect_ratio"], i["stretch_e"], i["principal_pt_x"], i["principal_pt_y"],
                                                          i["polynomial_a2"], i["polynomial_a3"], i["polynomial_a4"], i["stretch_d"]]
