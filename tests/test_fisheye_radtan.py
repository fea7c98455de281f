"""FISHEYE_RADIAL_TANGENTIAL (Kannala-Brandt with k1..k6 and tangential t1, t2; Fisheye62) on the CPU: the product's device math compiled
for the CPU and the NumPy model against OpenCV's own pixels (tests/golden/fisheye_radtan_opencv.npz), the reduction to FISHEYE at
k5 = k6 = t1 = t2 = 0, the closed-form Jacobians against central differences and the oracle-form autodiff (tests/fisheye_radtan/), the
limit at the optical axis, the domain rule against a dense scan, the unprojection and bearings, the camera calibration's rows, and the camera
JSON through both writers, the hot CLI's reader and the printed line."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from openimucameracalibrator_b200 import calibrator
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
GOLDEN = os.path.join(HERE, "golden", "fisheye_radtan_opencv.npz")
DP = ctypes.POINTER(ctypes.c_double)
FR, FISH = cm.FISHEYE_RADIAL_TANGENTIAL, cm.FISHEYE
NI = cm.MAX_INTRINSICS
# [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2]
K_WIDE = np.array([380.0, 1.003, 0.0, 640.5, 361.2, 0.05, -0.012, 0.003, -4e-4, 6e-5, -4e-6, 1.2e-3, -8e-4])    # monotone past 90 degrees
K_SKEW = np.array([420.0, 0.997, 0.4, 320.5, 240.2, -0.02, 0.01, -2e-3, 3e-4, -2e-5, 1e-6, -5e-4, 2e-3])
K_FOLD = np.array([400.0, 1.0, 0.0, 320.0, 240.0, -0.3, 0.0, 0.0, 0.0, 0.0, 0.0, 1e-3, -1e-3])               # d theta_d / d theta = 0 at theta^2 = 10/9
KS, KS_IDS = [K_WIDE, K_SKEW, K_FOLD], ["wide", "skew", "fold"]


def _dp(a):
    return a.ctypes.data_as(DP)


@pytest.fixture(scope="module")
def fhm(tmp_path_factory):
    """the product's __host__ __device__ camera math compiled for the CPU"""
    out = tmp_path_factory.mktemp("fisheye_radtan_hm") / "libfhm.so"
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets", "-o", str(out),
                           os.path.join(HERE, "fisheye_radtan", "fisheye_radtan_host_math.cu")])
    lib = ctypes.CDLL(str(out))
    lib.fhm_in_domain.argtypes = [DP, ctypes.c_double]
    lib.fhm_unproject.argtypes = [ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, DP]
    lib.fhm_bearing.argtypes = [ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, DP]
    return lib


@pytest.fixture(scope="module")
def oad(tmp_path_factory):
    """the oracle-form projection on dual numbers"""
    out = tmp_path_factory.mktemp("fisheye_radtan_oad") / "liboad.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(out), os.path.join(HERE, "fisheye_radtan", "oracle_autodiff_project.cpp")])
    return ctypes.CDLL(str(out))


def _kk(k):
    kk = np.zeros(NI); kk[: len(k)] = k
    return kk


def _project(fhm, model, k, p):
    out = np.zeros(8 + 2 * NI)
    rc = fhm.fhm_project(ctypes.c_int(model), _dp(_kk(k)), _dp(np.ascontiguousarray(p, dtype=np.float64)), _dp(out))
    assert rc & 2, "project() and project_with_k() disagree"
    return bool(rc & 1), out[:2].copy(), out[2:8].reshape(2, 3).copy(), out[8:].reshape(2, NI).copy()


def _golden_cases():
    z = np.load(GOLDEN)
    for i in range(int(z["n_cases"])):
        yield str(z[f"kind_{i}"]), z[f"K_{i}"], z[f"D_{i}"], z[f"T_{i}"], z[f"points_{i}"], z[f"xr_{i}"], z[f"uv_{i}"]


def _theia(K, D, T):
    return np.array([K[0, 0], K[1, 1] / K[0, 0], K[0, 1], K[0, 2], K[1, 2]] + list(D) + list(T))


def _theta_max(k):
    return min(cm.fisheye_radtan_theta_max(k), np.radians(85.0))


def _points(k, seed, n=200):
    """points in front of the camera with rays inside the domain (and below 85 degrees), with a margin of 1e-3 rad"""
    rng = np.random.default_rng(seed)
    th = rng.uniform(0.0, _theta_max(k) - 1e-3, n); ph = rng.uniform(0, 2 * np.pi, n); d = rng.uniform(0.3, 5.0, n)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1) * d[:, None]


def test_model_tables(fhm):
    assert fhm.fhm_c_enum() == fhm.fhm_device_enum() == FR == 10 and cm.MODEL_IDS["FISHEYE_RADIAL_TANGENTIAL"] == FR
    assert fhm.fhm_num_params(FR) == cm.NUM_PARAMS[FR] == cm.CAMERAS[FR].num_params == 13 == fhm.fhm_max_intrinsics() == NI
    keys = cm.CAMERAS[FR].keys
    assert [keys[f"radial_distortion_{i}"] for i in range(1, 7)] == list(range(5, 11))
    assert (keys["tangential_distortion_1"], keys["tangential_distortion_2"]) == (11, 12)


# ---- OpenCV's pixels ------------------------------------------------------------------------------------------------------------------
def test_product_and_numpy_reproduce_opencv_pixels(fhm):
    seen = set()
    for kind, K, D, T, P, xr, uv in _golden_cases():
        k = _theia(K, D, T)
        uvn, okn = cm.project(FR, k, P)
        assert okn.all() and np.abs(uvn - uv).max() < 1e-9, kind
        for p, ref in zip(P, uv):
            ok, px, _, _ = _project(fhm, FR, k, p)
            assert ok and np.abs(px - ref).max() < 1e-9, (kind, px, ref)
        seen.add(kind)
        if kind == "fisheye":
            assert np.degrees(np.arctan2(np.hypot(P[:, 0], P[:, 1]), P[:, 2])).max() > 85.0
    assert seen == {"fisheye", "tangential"}


def test_fixture_recomputes_with_cv2():
    pytest.importorskip("cv2")
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_fisheye_radtan_golden as mk
    golden = list(_golden_cases())
    assert len(golden) == len(mk.cases())
    for (kind, K, D, T, P), g in zip(mk.cases(), golden):
        assert kind == g[0] and np.array_equal(K, g[1]) and np.array_equal(D, g[2]) and np.array_equal(T, g[3]) and np.array_equal(P, g[4])
        uv, xr = mk.project(kind, K, D, T, P)
        assert np.abs(uv - g[6]).max() < 1e-9 and xr.shape == g[5].shape and np.abs(xr - g[5]).max(initial=0.0) <= 1e-15


# ---- reduction, derivatives ---------------------------------------------------------------------------------------------------------------
def _near_axis(seed, n=40):
    """points inside FISHEYE's own r^2 < 1e-8 branch at z = 1, the only depth where that branch's (x, y) is the projection's value"""
    rng = np.random.default_rng(seed)
    r = 10.0 ** rng.uniform(-9.0, -5.0, n); ph = rng.uniform(0, 2 * np.pi, n)
    return np.stack([r * np.cos(ph), r * np.sin(ph), np.ones(n)], -1)


@pytest.mark.parametrize("seed", [0, 1])
def test_reduced_model_is_fisheye(fhm, seed):
    k = K_WIDE.copy(); k[9:] = 0.0
    P = _points(k, seed, 150)
    for p in P:
        ok, px, Jp, Jk = _project(fhm, FR, k, p)
        ok1, px1, Jp1, Jk1 = _project(fhm, FISH, k[:9], p)
        assert ok and ok1
        assert np.abs(px - px1).max() <= 1e-12 * np.abs(px1).max()
        assert np.abs(Jp - Jp1).max() <= 1e-12 * np.abs(Jp1).max()
        assert np.abs(Jk[:, :9] - Jk1[:, :9]).max() <= 1e-12 * np.abs(Jk1).max()
    # inside FISHEYE's branch the values agree; its Jacobian drops d/dz and the 1/z of (x, y) / z, so they agree only as r -> 0
    for p in _near_axis(seed):
        ok, px, Jp, Jk = _project(fhm, FR, k, p)
        ok1, px1, Jp1, Jk1 = _project(fhm, FISH, k[:9], p)
        assert ok and ok1 and np.abs(px - px1).max() <= 1e-12 * np.abs(px1).max()
        r = np.hypot(p[0], p[1])
        assert np.abs(Jp - Jp1).max() <= (1e-12 + 2.0 * r) * np.abs(Jp1).max()
    for p in (np.array([0.0, 0.0, 1.0]), np.array([1e-15, -2e-15, 1.0])):
        ok, px, Jp, Jk = _project(fhm, FR, k, p)
        ok1, px1, Jp1, Jk1 = _project(fhm, FISH, k[:9], p)
        assert np.abs(px - px1).max() <= 1e-12 * np.abs(px1).max() and np.abs(Jp - Jp1).max() <= 1e-12 * np.abs(Jp1).max()
        assert np.abs(Jk[:, :9] - Jk1[:, :9]).max() <= 1e-12 * np.abs(Jk1).max()


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_jacobians_match_central_differences_and_autodiff(fhm, oad, k):
    for p in _points(k, 3, 40):
        ok, px, Jp, Jk = _project(fhm, FR, k, p)
        assert ok
        pa, Ja, Jka = np.zeros(2), np.zeros(6), np.zeros(2 * NI)
        oad.oad_fisheye_radtan_project(_dp(np.ascontiguousarray(k)), _dp(np.ascontiguousarray(p)), _dp(pa), _dp(Ja), _dp(Jka))
        assert np.abs(pa - px).max() < 1e-9
        assert np.abs(Ja.reshape(2, 3) - Jp).max() <= 1e-10 * max(1.0, np.abs(Jp).max())
        assert np.abs(Jka.reshape(2, NI) - Jk).max() <= 1e-10 * max(1.0, np.abs(Jk).max())
        for j in range(3):
            h = 1e-6 * max(1.0, abs(p[j]))
            e = np.zeros(3); e[j] = h
            num = (_project(fhm, FR, k, p + e)[1] - _project(fhm, FR, k, p - e)[1]) / (2 * h)
            assert np.abs(num - Jp[:, j]).max() <= 1e-5 * max(1.0, np.abs(Jp).max())
        for q in range(NI):
            h = 1e-6 * max(1.0, abs(k[q]))
            e = np.zeros(NI); e[q] = h
            num = (_project(fhm, FR, k + e, p)[1] - _project(fhm, FR, k - e, p)[1]) / (2 * h)
            assert np.abs(num - Jk[:, q]).max() <= 1e-5 * max(1.0, np.abs(Jk).max()), q


def test_limit_at_the_optical_axis(fhm):
    """finite values and Jacobians at theta = 0, continuous over theta in [1e-12, 1e-6] (across the series branch at a^2 = 1e-8) and on to
    theta = 1e-3"""
    k = K_SKEW
    for z, ph in ((1.0, 0.3), (2.5, 2.0), (0.4, -1.1)):
        ok0, px0, J0, Jk0 = _project(fhm, FR, k, np.array([0.0, 0.0, z]))
        assert ok0 and np.isfinite(J0).all() and np.isfinite(Jk0).all()
        # on the axis: the pinhole at the principal point, d(u, v)/d(x, y) = f [[1, skew / f], [0, ar]] / z
        assert np.array_equal(px0, k[3:5]) and np.allclose(J0[:, :2], np.array([[k[0], k[2]], [0.0, k[0] * k[1]]]) / z, rtol=1e-15, atol=0)
        prev = None
        for th in np.concatenate([10.0 ** np.linspace(-12, -6, 61), [1e-3]]):
            p = z * np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
            ok, px, Jp, Jk = _project(fhm, FR, k, p)
            assert ok and np.isfinite(Jp).all() and np.isfinite(Jk).all()
            if th <= 1e-6:           # within O(theta) of the axis values
                assert np.abs(Jp - J0).max() <= 4.0 * th * np.abs(J0).max() and np.abs(px - px0).max() <= 2.0 * k[0] * th
            if prev is not None:
                assert np.abs(Jp - prev).max() <= 10.0 * th * np.abs(J0).max()
            prev = Jp


def test_axis_branch_matches_autodiff_just_outside_it(fhm, oad):
    """a^2 = r^2 / z^2 on both sides of the series branch's edge 1e-8: the closed form against the Jet statement"""
    for a in (0.9e-4, 0.99999e-4, 1.00001e-4, 1.1e-4, 3e-4):
        for z in (0.5, 1.0, 3.0):
            p = np.array([0.6 * a * z, 0.8 * a * z, z])
            ok, px, Jp, Jk = _project(fhm, FR, K_SKEW, p)
            pa, Ja, Jka = np.zeros(2), np.zeros(6), np.zeros(2 * NI)
            oad.oad_fisheye_radtan_project(_dp(np.ascontiguousarray(K_SKEW)), _dp(p), _dp(pa), _dp(Ja), _dp(Jka))
            assert ok and np.abs(pa - px).max() <= 1e-12 * np.abs(px).max()
            assert np.abs(Ja.reshape(2, 3) - Jp).max() <= 1e-12 * np.abs(Jp).max()
            assert np.abs(Jka.reshape(2, NI) - Jk).max() <= 1e-12 * np.abs(Jk).max()


# ---- domain, unprojection -------------------------------------------------------------------------------------------------------------
def _scan_theta_max(k, th_hi=3.0, n=3_000_001):
    th = np.linspace(0.0, th_hi, n); t = th * th
    thd = th * (1 + t * (k[5] + t * (k[6] + t * (k[7] + t * (k[8] + t * (k[9] + t * k[10]))))))
    bad = np.diff(thd) <= 0.0
    return (th[1:][bad][0], th[1] - th[0]) if bad.any() else (np.inf, th[1] - th[0])


@pytest.mark.parametrize("k", KS + [np.array([400.0, 1, 0, 320, 240, 0.1, -0.2, 0.05, 0.0, 0.0, -0.01, 0.0, 0.0])], ids=KS_IDS + ["k6_fold"])
def test_domain_matches_a_dense_scan_and_the_device_rule(fhm, k):
    thmax = cm.fisheye_radtan_theta_max(k)
    scan, dth = _scan_theta_max(k)
    assert (np.isinf(thmax) and np.isinf(scan)) or abs(min(thmax, 3.0) - min(scan, 3.0)) <= 2 * dth or (thmax > 3.0 and np.isinf(scan))
    kk = _kk(k)
    grid = np.linspace(0.0, np.pi / 2, 2001)[1:]
    for th in grid[np.abs(grid - thmax) > 1e-6 * max(1.0, thmax)]:
        assert bool(fhm.fhm_in_domain(_dp(kk), th * th)) == (th < thmax), th
        p = np.array([np.sin(th), 0.0, np.cos(th)])
        if p[2] > 0.0:
            assert _project(fhm, FR, k, p)[0] == (th < thmax) == cm.project(FR, k, p[None])[1][0]
    if thmax < np.pi / 2:
        assert fhm.fhm_in_domain(_dp(kk), (thmax * (1 - 1e-9)) ** 2) and not fhm.fhm_in_domain(_dp(kk), (thmax * (1 + 1e-9)) ** 2)


def test_points_behind_the_camera_fail(fhm):
    for p in ([0.1, 0.2, -1.0], [0.0, 0.0, 0.0], [0.3, -0.1, -1e-9], [1.0, 0.0, 0.0], [0.0, 0.0, -2.0]):
        ok, px, Jp, Jk = _project(fhm, FR, K_WIDE, np.array(p))
        assert not ok and not px.any() and not Jp.any() and not Jk.any()
        assert not cm.project(FR, K_WIDE, np.array([p]))[1][0]


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_unprojection_and_bearings_invert_the_projection(fhm, k):
    P = _points(k, 5, 100)
    uv, ok = cm.project(FR, k, P)
    assert ok.all()
    xy_np, ok_np = cm.fisheye_radtan_unproject(k, uv)
    assert ok_np.all()
    kk = _kk(k)
    for p, q, xyn in zip(P, uv, xy_np):
        xy, b = np.zeros(2), np.zeros(3)
        assert fhm.fhm_unproject(FR, _dp(kk), q[0], q[1], _dp(xy))
        assert fhm.fhm_bearing(FR, _dp(kk), q[0], q[1], _dp(b))
        assert np.abs(cm.project(FR, k, np.array([[xy[0], xy[1], 1.0]]))[0][0] - q).max() < 1e-9
        assert np.abs(cm.project(FR, k, np.array([[xyn[0], xyn[1], 1.0]]))[0][0] - q).max() < 1e-9
        assert np.abs(cm.project(FR, k, b[None])[0][0] - q).max() < 1e-9 and b[2] > 0.0
        assert np.abs(b - p / np.linalg.norm(p)).max() < 1e-8


def test_camera_calibration_rows_carry_all_thirteen_columns(fhm):
    X = np.array([0.4, -0.25, 1.5]); q = np.array([0.0, 0.0, 0.0, 1.0]); c = np.zeros(3); uv = np.array([700.0, 300.0])
    r, J0, J1 = np.zeros(2), np.zeros(NI), np.zeros(NI)
    assert fhm.fhm_camcal_rows(FR, _dp(K_WIDE), _dp(q), _dp(c), _dp(X), _dp(uv), _dp(r), _dp(J0), _dp(J1))
    ok, px, _, Jk = _project(fhm, FR, K_WIDE, X)
    assert np.array_equal(r, px - uv) and np.array_equal(J0, Jk[0]) and np.array_equal(J1, Jk[1]) and np.abs(Jk[:, 10:]).min() > 0


# ---- formats -----------------------------------------------------------------------------------------------------------------------------
def _parse_only(paths, tmp_path):
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/result.json", f"--output_path={tmp_path}", "--parse_only"]
    return subprocess.run(args, capture_output=True, text=True)


def test_cli_reads_the_written_camera(tmp_path):
    paths = iof.write_dataset_files(syn.make_dataset(syn.tiny_config(FR, tuple(K_SKEW), n_frames=8)), str(tmp_path))
    cam = json.load(open(paths["camera_calibration_json"]))
    i = cam["intrinsics"]
    assert cam["intrinsic_type"] == "FISHEYE_RADIAL_TANGENTIAL" and i["radial_distortion_5"] == K_SKEW[9] and i["radial_distortion_6"] == K_SKEW[10]
    assert (i["tangential_distortion_1"], i["tangential_distortion_2"]) == (K_SKEW[11], K_SKEW[12])
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    expect = K_SKEW.copy(); expect[2] = 0.0                                    # the skew is never read
    assert s["camera_model"] == FR and np.array_equal(np.array(s["intrinsics"]), expect)
    del cam["intrinsics"]["tangential_distortion_2"]
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode != 0 and "missing key 'tangential_distortion_2'" in out.stderr


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("fisheye_radtan_json") / "camera_json_shim")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-o", out, os.path.join(HERE, "camera_json", "camera_json_shim.cpp")])
    return lambda *a: subprocess.run([out, *a], capture_output=True, text=True)


def test_cpp_writer_and_printed_line(shim, monkeypatch, capsys):
    k = K_WIDE.copy(); k[2] = 0.0
    out = shim("write", "FISHEYE_RADIAL_TANGENTIAL", *map(repr, map(float, k)))
    assert out.returncode == 0, out.stderr
    assert json.loads(out.stdout) == iof.intrinsics_dict(FR, k) == dict(
        focal_length=k[0], aspect_ratio=k[1], skew=0.0, principal_pt_x=k[3], principal_pt_y=k[4], **{f"radial_distortion_{j}": k[4 + j] for j in range(1, 7)},
        tangential_distortion_1=k[11], tangential_distortion_2=k[12])
    line = ("FISHEYE_RADIAL_TANGENTIAL model: " + " ".join(f"Radial distortion {j}: {{{4 + j}}}" for j in range(1, 7)) +
            " Tangential distortion 1: {11} Tangential distortion 2: {12}")
    monkeypatch.setattr(calibrator, "load_library", lambda: None)
    monkeypatch.setattr(calibrator, "CApi", lambda *a: None)
    cal = calibrator.CameraCalibrator("FISHEYE_RADIAL_TANGENTIAL")
    cal.result = {"intrinsics": k}
    cal.PrintResult()
    assert capsys.readouterr().out == f"Focal Length:{k[0]}px Principal Point: {k[3]}/{k[4]}px.\n" + line.format(*k) + "\n"
    out = shim("print", "FISHEYE_RADIAL_TANGENTIAL", *map(repr, map(float, k)))
    assert out.returncode == 0 and out.stdout.splitlines()[1] == line.format(*(format(v, "g") for v in k))
