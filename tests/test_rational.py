"""PINHOLE_RATIONAL (OpenCV's rational polynomial model, k1..k6, p1, p2) on the CPU: the product's device math compiled for the CPU and the
NumPy model against cv2.projectPoints' own pixels (tests/golden/rational_opencv_projectpoints.npz), the reduction to
PINHOLE_RADIAL_TANGENTIAL at k4 = k5 = k6 = 0, the closed-form Jacobians against central differences and the oracle-form autodiff
(tests/rational/), the domain rule and its s_max against a dense scan, the unprojection, the camera JSON through both writers' readers,
and the OpenCV / ROS importer."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import opencv_to_json as o2j
from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
GOLDEN = os.path.join(HERE, "golden", "rational_opencv_projectpoints.npz")
DP = ctypes.POINTER(ctypes.c_double)
RAT, RADTAN = cm.PINHOLE_RATIONAL, cm.PINHOLE_RADIAL_TANGENTIAL
NI = cm.MAX_INTRINSICS
# [f, ar, skew, cx, cy, k1, k2, k3, t1, t2, k4, k5, k6]
K_WIDE = np.array([610.0, 1.004, 0.0, 641.0, 359.0, 0.35, -0.08, 0.004, 1.2e-3, -8e-4, 0.72, -0.02, 0.01])      # s_max = 1.96 (54 degrees)
K_SKEW = np.array([480.0, 0.997, 0.4, 320.5, 240.2, -0.2, 0.05, -0.003, -4e-4, 7e-4, 0.1, 0.02, -0.001])
K_POLE = np.array([500.0, 1.0, 0.0, 320.0, 240.0, 0.1, 0.0, 0.0, 0.0, 0.0, -0.5, 0.0, 0.0])                   # M = 0 at s = 2
KS, KS_IDS = [K_WIDE, K_SKEW, K_POLE], ["wide", "skew", "pole"]


def _dp(a):
    return a.ctypes.data_as(DP)


@pytest.fixture(scope="module")
def rhm(tmp_path_factory):
    """the product's __host__ __device__ camera math compiled for the CPU"""
    out = tmp_path_factory.mktemp("rational_hm") / "librhm.so"
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets", "-o", str(out),
                           os.path.join(HERE, "rational", "rational_host_math.cu")])
    lib = ctypes.CDLL(str(out))
    lib.rhm_in_domain.argtypes = [DP, ctypes.c_double]
    lib.rhm_unproject.argtypes = [ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, DP]
    lib.rhm_bearing.argtypes = [ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, DP]
    return lib


@pytest.fixture(scope="module")
def oad(tmp_path_factory):
    """the oracle-form projection on dual numbers"""
    out = tmp_path_factory.mktemp("rational_oad") / "liboad.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(out), os.path.join(HERE, "rational", "oracle_autodiff_project.cpp")])
    return ctypes.CDLL(str(out))


def _kk(k):
    kk = np.zeros(NI); kk[: len(k)] = k
    return kk


def _project(rhm, model, k, p):
    out = np.zeros(8 + 2 * NI)
    rc = rhm.rhm_project(ctypes.c_int(model), _dp(_kk(k)), _dp(np.ascontiguousarray(p, dtype=np.float64)), _dp(out))
    assert rc & 2, "project() and project_with_k() disagree"
    return bool(rc & 1), out[:2].copy(), out[2:8].reshape(2, 3).copy(), out[8:].reshape(2, NI).copy()


def _golden_cases():
    z = np.load(GOLDEN)
    for i in range(int(z["n_cases"])):
        yield str(z[f"kind_{i}"]), z[f"K_{i}"], z[f"D_{i}"], z[f"points_{i}"], z[f"uv_{i}"]


def _theia(kind, K, D):
    head = [K[0, 0], K[1, 1] / K[0, 0], K[0, 1], K[0, 2], K[1, 2]]
    if kind == "fisheye":
        return cm.FISHEYE, np.array(head + list(D))
    return RAT, np.array(head + [D[0], D[1], D[4], D[2], D[3], D[5], D[6], D[7]])


def _points(k, seed, n=300):
    """points in front of the camera, inside the domain with a margin of 1e-3 in s"""
    rng = np.random.default_rng(seed)
    smax = min(cm.rational_s_max(k), 9.0)
    s = rng.uniform(0.0, smax - 1e-3, n); ph = rng.uniform(0, 2 * np.pi, n); z = rng.uniform(0.3, 5.0, n)
    r = np.sqrt(s)
    return np.stack([r * np.cos(ph) * z, r * np.sin(ph) * z, z], -1)


def test_model_tables(rhm):
    assert rhm.rhm_max_intrinsics() == NI == 13 and rhm.rhm_num_params(RAT) == cm.NUM_PARAMS[RAT] == 13
    assert cm.MODEL_IDS["PINHOLE_RATIONAL"] == RAT == 9 and max(cm.NUM_PARAMS.values()) == NI


# ---- OpenCV's pixels ------------------------------------------------------------------------------------------------------------------
def test_product_and_numpy_reproduce_opencv_pixels(rhm):
    for kind, K, D, P, uv in _golden_cases():
        model, k = _theia(kind, K, D)
        uvn, okn = cm.project(model, k, P)
        assert okn.all() and np.abs(uvn - uv).max() < 1e-9, kind
        for p, ref in zip(P, uv):
            ok, px, _, _ = _project(rhm, model, k, p)
            assert ok and np.abs(px - ref).max() < 1e-9, (kind, px, ref)


def test_fixture_recomputes_with_cv2():
    pytest.importorskip("cv2")
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_rational_golden as mk
    golden = list(_golden_cases())
    for (kind, K, D, P), g in zip(mk.cases(), golden):
        assert kind == g[0] and np.array_equal(K, g[1]) and np.array_equal(D, g[2]) and np.array_equal(P, g[3])
        assert np.abs(mk.project(kind, K, D, P) - g[4]).max() < 1e-9


# ---- reduction, derivatives ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_zero_denominator_is_the_radial_tangential_model(rhm, seed):
    k = K_SKEW.copy(); k[10:] = 0.0
    for p in _points(k, seed, 100):
        ok, px, Jp, Jk = _project(rhm, RAT, k, p)
        ok1, px1, Jp1, Jk1 = _project(rhm, RADTAN, k[:10], p)
        assert ok and ok1
        scale = max(np.abs(px1).max(), 1.0)
        assert np.abs(px - px1).max() <= 1e-14 * scale
        assert np.abs(Jp - Jp1).max() <= 1e-14 * np.abs(Jp1).max()
        assert np.abs(Jk[:, :10] - Jk1[:, :10]).max() <= 1e-14 * np.abs(Jk1).max()


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_jacobians_match_central_differences_and_autodiff(rhm, oad, k):
    for p in _points(k, 3, 40):
        ok, px, Jp, Jk = _project(rhm, RAT, k, p)
        assert ok
        pa, Ja, Jka = np.zeros(2), np.zeros(6), np.zeros(2 * NI)
        oad.oad_rational_project(_dp(np.ascontiguousarray(k)), _dp(np.ascontiguousarray(p)), _dp(pa), _dp(Ja), _dp(Jka))
        assert np.abs(pa - px).max() < 1e-9
        assert np.abs(Ja.reshape(2, 3) - Jp).max() <= 1e-10 * max(1.0, np.abs(Jp).max())
        assert np.abs(Jka.reshape(2, NI) - Jk).max() <= 1e-10 * max(1.0, np.abs(Jk).max())
        for j in range(3):
            h = 1e-6 * max(1.0, abs(p[j]))
            e = np.zeros(3); e[j] = h
            num = (_project(rhm, RAT, k, p + e)[1] - _project(rhm, RAT, k, p - e)[1]) / (2 * h)
            assert np.abs(num - Jp[:, j]).max() <= 1e-5 * max(1.0, np.abs(Jp).max())
        for q in range(NI):
            h = 1e-6 * max(1.0, abs(k[q]))
            e = np.zeros(NI); e[q] = h
            num = (_project(rhm, RAT, k + e, p)[1] - _project(rhm, RAT, k - e, p)[1]) / (2 * h)
            assert np.abs(num - Jk[:, q]).max() <= 1e-5 * max(1.0, np.abs(Jk).max()), q


# ---- domain, unprojection -------------------------------------------------------------------------------------------------------------
def _scan_s_max(k, s_hi=12.0, n=2_400_001):
    s = np.linspace(0.0, s_hi, n)
    N = 1 + s * (k[5] + s * (k[6] + s * k[7])); M = 1 + s * (k[10] + s * (k[11] + s * k[12]))
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.sqrt(s) * N / M
    bad = (np.diff(f) <= 0.0) | (M[1:] <= 0.0)
    return (s[1:][bad][0], s[1] - s[0]) if bad.any() else (np.inf, s[1] - s[0])


@pytest.mark.parametrize("k", KS + [np.array([500.0, 1, 0, 320, 240, -0.3, 0.1, -0.01, 0, 0, 0.1, 0.02, 0.0]),
                                    np.array([500.0, 1, 0, 320, 240, 0.5, 0.0, 0.0, 0, 0, 0.9, 0.3, 0.1])],
                         ids=KS_IDS + ["fold", "flat_denominator"])
def test_s_max_matches_a_dense_scan_and_the_device_rule(rhm, k):
    smax = cm.rational_s_max(k)
    scan, ds = _scan_s_max(k)
    assert (np.isinf(smax) and np.isinf(scan)) or abs(smax - scan) <= 2 * ds
    kk = _kk(k)
    grid = np.linspace(0.0, 12.0, 4001)[1:]
    for s in grid[np.abs(grid - smax) > 1e-6 * max(1.0, smax)]:
        assert bool(rhm.rhm_in_domain(_dp(kk), s)) == (s < smax), s
    if np.isfinite(smax):
        assert rhm.rhm_in_domain(_dp(kk), smax * (1 - 1e-9)) and not rhm.rhm_in_domain(_dp(kk), smax * (1 + 1e-9))
        # a point past s_max fails in both statements
        p = np.array([np.sqrt(smax * 1.01), 0.0, 1.0])
        assert not _project(rhm, RAT, k, p)[0] and not cm.project(RAT, k, p[None])[1][0]


def test_points_behind_the_camera_and_on_a_negative_denominator_fail(rhm):
    for p in ([0.1, 0.2, -1.0], [0.0, 0.0, 0.0], [0.3, -0.1, -1e-9]):
        ok, px, Jp, Jk = _project(rhm, RAT, K_WIDE, np.array(p))
        assert not ok and not px.any() and not Jp.any() and not Jk.any()
        assert not cm.project(RAT, K_WIDE, np.array([p]))[1][0]
    p = np.array([np.sqrt(2.5), 0.0, 1.0])              # K_POLE: M(2.5) = -0.25
    assert not _project(rhm, RAT, K_POLE, p)[0] and not cm.project(RAT, K_POLE, p[None])[1][0]


@pytest.mark.parametrize("k", KS, ids=KS_IDS)
def test_unprojection_inverts_the_projection(rhm, k):
    P = _points(k, 5, 100)
    uv, ok = cm.project(RAT, k, P)
    assert ok.all()
    xy_np, ok_np = cm.rational_unproject(k, uv)
    assert ok_np.all()
    kk = _kk(k)
    for p, q, xyn in zip(P, uv, xy_np):
        xy, b = np.zeros(2), np.zeros(3)
        assert rhm.rhm_unproject(RAT, _dp(kk), q[0], q[1], _dp(xy))
        assert rhm.rhm_bearing(RAT, _dp(kk), q[0], q[1], _dp(b))
        back = cm.project(RAT, k, np.array([[xy[0], xy[1], 1.0]]))[0][0]
        assert np.abs(back - q).max() < 1e-9
        assert np.abs(cm.project(RAT, k, np.array([[xyn[0], xyn[1], 1.0]]))[0][0] - q).max() < 1e-9
        assert np.abs(cm.project(RAT, k, b[None])[0][0] - q).max() < 1e-9
        if (p[0] ** 2 + p[1] ** 2) / p[2] ** 2 < 0.8 * min(cm.rational_s_max(k), 9.0):   # next to the fold the tangential terms may fold the image too
            assert np.abs(b - p / np.linalg.norm(p)).max() < 1e-9


def test_bearing_of_a_pixel_beyond_the_fold_is_refused(rhm):
    k = K_WIDE
    smax = cm.rational_s_max(k)
    edge = cm.project(RAT, k, np.array([[np.sqrt(smax) * (1 - 1e-6), 0.0, 1.0]]))[0][0]
    far = k[3] + 1.05 * (edge[0] - k[3])                # past the largest radius the lens reaches along +x
    b = np.zeros(3)
    assert not rhm.rhm_bearing(RAT, _dp(_kk(k)), far, k[4], _dp(b))
    assert not cm.rational_unproject(k, np.array([[far, k[4]]]))[1][0]


def test_camera_calibration_rows_carry_all_thirteen_columns(rhm):
    X = np.array([0.1, -0.05, 1.5]); q = np.array([0.0, 0.0, 0.0, 1.0]); c = np.zeros(3); uv = np.array([600.0, 340.0])
    r, J0, J1 = np.zeros(2), np.zeros(NI), np.zeros(NI)
    assert rhm.rhm_camcal_rows(RAT, _dp(K_WIDE), _dp(q), _dp(c), _dp(X), _dp(uv), _dp(r), _dp(J0), _dp(J1))
    ok, px, _, Jk = _project(rhm, RAT, K_WIDE, X)
    assert np.array_equal(r, px - uv) and np.array_equal(J0, Jk[0]) and np.array_equal(J1, Jk[1]) and np.abs(Jk[:, 10:]).min() > 0


# ---- formats -----------------------------------------------------------------------------------------------------------------------------
def _tiny(k=K_WIDE, **kw):
    return syn.tiny_config(RAT, tuple(k), **kw)


def _parse_only(paths, tmp_path):
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/result.json", f"--output_path={tmp_path}", "--parse_only"]
    return subprocess.run(args, capture_output=True, text=True)


def test_cli_reads_the_written_camera(tmp_path):
    paths = iof.write_dataset_files(syn.make_dataset(_tiny(n_frames=8)), str(tmp_path))
    cam = json.load(open(paths["camera_calibration_json"]))
    assert cam["intrinsic_type"] == "PINHOLE_RATIONAL" and cam["intrinsics"]["radial_distortion_4"] == K_WIDE[10] and cam["intrinsics"]["radial_distortion_6"] == K_WIDE[12]
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == RAT and np.array_equal(np.array(s["intrinsics"]), K_WIDE)
    del cam["intrinsics"]["radial_distortion_5"]
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode != 0 and "missing key 'radial_distortion_5'" in out.stderr


# ---- importer ----------------------------------------------------------------------------------------------------------------------------
def _opencv_yaml(K, D, W=1280, H=720, names=("camera_matrix", "distortion_coefficients"), extra=""):
    def mat(name, rows, cols, data):
        vals = [repr(float(v)) for v in data]         # the list over two lines, as cv2.FileStorage writes long ones
        h = len(vals) // 2
        return f"{name}: !!opencv-matrix\n   rows: {rows}\n   cols: {cols}\n   dt: d\n   data: [ {', '.join(vals[:h])},\n       {', '.join(vals[h:])} ]\n"
    return f"%YAML:1.0\n---\nimage_width: {W}\nimage_height: {H}\n" + mat(names[0], 3, 3, np.ravel(K)) + mat(names[1], 1, len(D), D) + extra


def _ros_yaml(K, D, model, W=1280, H=720):
    return (f"image_width: {W}\nimage_height: {H}\ncamera_name: cam0  # a comment\ncamera_matrix:\n  rows: 3\n  cols: 3\n  data: [{', '.join(map(repr, map(float, np.ravel(K))))}]\n"
            f"distortion_model: {model}\ndistortion_coefficients:\n  rows: 1\n  cols: {len(D)}\n  data: [{', '.join(map(repr, map(float, D)))}]\n"
            "rectification_matrix:\n  rows: 3\n  cols: 3\n  data: [1, 0, 0, 0, 1, 0, 0, 0, 1]\n")


def _opencv_json(K, D, W=1280, H=720):
    m = lambda r, c, d: {"type_id": "opencv-matrix", "rows": r, "cols": c, "dt": "d", "data": [float(v) for v in np.ravel(d)]}   # noqa: E731
    return json.dumps({"image_width": W, "image_height": H, "camera_matrix": m(3, 3, K), "distortion_coefficients": m(1, len(D), D)})


def _import(tmp_path, text, *extra):
    src, dst = tmp_path / "calib.in", tmp_path / "cam.json"
    src.write_text(text)
    return o2j.main(["--input", str(src), "--output", str(dst), "--fps", "30", *extra]), dst


def _product_pixels(rhm, doc, P):
    i = doc["intrinsics"]
    model = cm.MODEL_IDS[doc["intrinsic_type"]]
    head = [i["focal_length"], i["aspect_ratio"], i["skew"], i["principal_pt_x"], i["principal_pt_y"]]
    if model == RAT:
        k = head + [i[f"radial_distortion_{j}"] for j in (1, 2, 3)] + [i["tangential_distortion_1"], i["tangential_distortion_2"]] + [i[f"radial_distortion_{j}"] for j in (4, 5, 6)]
    elif model == cm.FISHEYE:
        k = head + [i[f"radial_distortion_{j}"] for j in (1, 2, 3, 4)]
    else:
        k = head + [i[f"radial_distortion_{j}"] for j in (1, 2, 3)] + [i["tangential_distortion_1"], i["tangential_distortion_2"]]
    return np.array([_project(rhm, model, k, p)[1] for p in P])


@pytest.mark.parametrize("fmt", ["opencv_yaml", "opencv_json", "ros", "opencv_yaml_KD", "ros_14"])
def test_importer_reproduces_opencv_pixels(rhm, tmp_path, fmt):
    for kind, K, D, P, uv in _golden_cases():
        if kind == "fisheye":
            continue
        text = {"opencv_yaml": lambda: _opencv_yaml(K, D), "opencv_json": lambda: _opencv_json(K, D), "ros": lambda: _ros_yaml(K, D, "rational_polynomial"),
                "opencv_yaml_KD": lambda: _opencv_yaml(K, D, names=("K", "D")), "ros_14": lambda: _ros_yaml(K, list(D) + [0.0] * 6, "rational_polynomial")}[fmt]()
        doc, dst = _import(tmp_path, text)
        assert doc["intrinsic_type"] == "PINHOLE_RATIONAL" and json.load(open(dst)) == doc and (doc["image_width"], doc["image_height"]) == (1280, 720)
        assert np.abs(_product_pixels(rhm, doc, P) - uv).max() < 1e-9


def test_importer_maps_five_coefficients_and_fisheye(rhm, tmp_path):
    K = np.array([[500.0, 0.0, 320.0], [0.0, 505.0, 240.0], [0.0, 0.0, 1.0]])
    for D in ([0.1, -0.02, 1e-3, 2e-3, 0.005], [0.1, -0.02, 1e-3, 2e-3]):
        doc, _ = _import(tmp_path, _ros_yaml(K, D, "plumb_bob"))
        assert doc["intrinsic_type"] == "PINHOLE_RADIAL_TANGENTIAL"
        i = doc["intrinsics"]
        assert [i["radial_distortion_1"], i["radial_distortion_2"], i["radial_distortion_3"], i["tangential_distortion_1"], i["tangential_distortion_2"]] == \
               [D[0], D[1], D[4] if len(D) == 5 else 0.0, D[2], D[3]]
    fish = [g for g in _golden_cases() if g[0] == "fisheye"][0]
    for text in (_ros_yaml(fish[1], fish[2], "equidistant"), _opencv_yaml(fish[1], fish[2], extra="fisheye_model: 1\n")):
        doc, _ = _import(tmp_path, text)
        assert doc["intrinsic_type"] == "FISHEYE"
        assert np.abs(_product_pixels(rhm, doc, fish[3]) - fish[4]).max() < 1e-9


def test_importer_takes_the_image_size_from_the_command_line(tmp_path):
    K, D = np.eye(3) * 400.0, [0.0] * 8
    K[2, 2] = 1.0
    doc, _ = _import(tmp_path, _opencv_yaml(K, D), "--width", "640", "--height", "480")
    assert (doc["image_width"], doc["image_height"]) == (640, 480)
    text = _opencv_yaml(K, D).replace("image_width: 1280\nimage_height: 720\n", "")
    with pytest.raises(SystemExit, match="no image size"):
        _import(tmp_path, text)


@pytest.mark.parametrize("D,msg", [([0.1] * 8 + [0.0, 2e-3, 0.0, 0.0], "s2 = 0.002"),
                                   ([0.1] * 8 + [0.0] * 4 + [0.0, 1e-4], "ty = 0.0001"),
                                   ([0.1] * 6, "6 distortion coefficients")])
def test_importer_refuses_what_the_models_cannot_hold(tmp_path, D, msg):
    K = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])
    with pytest.raises(SystemExit, match=msg):
        _import(tmp_path, _ros_yaml(K, D, "rational_polynomial"))
    assert not (tmp_path / "cam.json").exists()
    out = subprocess.run([sys.executable, "-m", "openimucameracalibrator_b200.opencv_to_json", "--input", str(tmp_path / "calib.in"), "--output",
                          str(tmp_path / "cam.json"), "--fps", "30"], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode != 0 and msg in out.stderr and not (tmp_path / "cam.json").exists()


def test_cli_reads_the_imported_camera(tmp_path):
    kind, K, D, P, uv = next(iter(_golden_cases()))
    paths = iof.write_dataset_files(syn.make_dataset(_tiny(n_frames=8)), str(tmp_path / "seq"))
    src = tmp_path / "calib.yaml"; src.write_text(_opencv_yaml(K, D))
    paths["camera_calibration_json"] = str(tmp_path / "cam.json")
    doc = o2j.main(["--input", str(src), "--output", paths["camera_calibration_json"], "--fps", "30"])
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == RAT and np.allclose(s["intrinsics"], _theia(kind, K, D)[1], rtol=0, atol=0) and doc["intrinsic_type"] == "PINHOLE_RATIONAL"
