"""The drop-in extract_board_to_json on the GPU: the colour entry against the gray entry on OpenCV's own resize + BGR2GRAY, then folders
of tinted PNG renders through the CLI (file layout, corners bit-identical to the entry, independence of the chunking, gray and colour
frames mixed) and on through calibrate_camera."""
import json
import os
import subprocess

import numpy as np
import pytest

import png_support as ps
from openimucameracalibrator_b200 import calibrator, camera_models as cm, io_formats, synthetic as syn
from openimucameracalibrator_b200._capi import CApi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")
W, H, SQ = 14, 9, 0.0121
SIZE = (1280, 720)
FACTOR = 2.0
# (calibrate_camera model name, render model, intrinsics, distances in m)
CAMERAS = {
    "pinhole": ("PINHOLE", cm.PINHOLE, (900.0, 1.0, 0.0, 641.0, 357.0, 0.0, 0.0), 0.26),
    "fisheye": ("FISHEYE", cm.FISHEYE, (460.0, 1.0, 0.0, 636.0, 362.0, 0.05, 0.07, -0.11, 0.05), 0.15),
}
TINT = ((0.6, 30.0), (0.9, 10.0), (0.7, 45.0))   # (gain, offset) of B, G, R on the gray render


@pytest.fixture(scope="module")
def api():
    return CApi(calibrator.load_library(), "icc_", 0)


def test_bgr_entry_equals_gray_entry_on_opencv_gray(api):
    import torch
    g = np.load(os.path.join(HERE, "golden", "bgr_resize_gray_opencv.npz"))
    bgr = g["bgr"]
    for f in (1.0, 1.5, 2.0, 3.0):
        gray = g["gray_" + f"{f:g}".replace(".", "p")]
        ref, fref, sref = api.extract_radon_board(gray, W, H, 1.0)
        uv, found, s = api.extract_radon_board_bgr(bgr, W, H, f)
        np.testing.assert_array_equal(found, fref)
        np.testing.assert_array_equal(uv, ref)
        assert (s["width"], s["height"]) == (sref["width"], sref["height"]) == gray.shape[2:0:-1]
        uvd, foundd, _ = api.extract_radon_board_bgr(torch.from_numpy(bgr).cuda(), W, H, f)
        np.testing.assert_array_equal(foundd, fref)
        np.testing.assert_array_equal(uvd, ref)
        if f == 1.0:
            assert found.all()


def _stamps(n):
    """Irregular stamps [ns]: 40 ms and 33.3 ms in turn, then one long interval, so that leaving out the last interval (the reference's
    loop bound) moves the median from 40 ms to the mean of the two."""
    dt = np.where(np.arange(n - 1) % 2, 33_333_333, 40_000_000).astype(np.int64)
    dt[-1] = 90_000_000
    return 1_700_000_000_000_000_000 + np.concatenate([[0], np.cumsum(dt)])


def _frames(name, n):
    _, model, intr, dist = CAMERAS[name]
    rng = np.random.default_rng(5 if name == "pinhole" else 6)
    out, has_board = [], []
    for k in range(n):
        empty = k in (4, 13)
        tilt, axis, roll = rng.uniform(5, 38), rng.uniform(0, 360), rng.uniform(-25, 25)
        off = (3.0, 0.0) if empty else tuple(rng.uniform(-0.012, 0.012, 2))
        R, t = syn.radon_view_pose(W, H, SQ, dist * rng.uniform(0.95, 1.1), tilt, axis, roll, offset_m=off)
        g, _, valid = syn.render_radon_board(model, intr, SIZE, R, t, W, H, SQ, supersample=2, blur_sigma_px=0.7, noise_sigma_dn=1.0, seed=k)
        ramp = np.linspace(-15, 15, SIZE[0])[None, :]
        bgr = np.stack([np.clip(a * g + b + s * ramp, 0, 255) for (a, b), s in zip(TINT, (1, 0, -1))], -1)
        out.append(np.rint(bgr).astype(np.uint8))
        has_board.append(not empty and bool(valid.all()))
    return out, has_board


@pytest.fixture(scope="module")
def folders(tmp_path_factory):
    """Per camera: ~20 frames written as <ns>.png, three of them as gray PNGs (the gray of the colour render), and the frames as
    decoded (BGR; the gray ones replicated)."""
    out = {}
    for name in CAMERAS:
        d = tmp_path_factory.mktemp(name)
        frames, has_board = _frames(name, 20)
        stamps = _stamps(len(frames))
        decoded = []
        for k, (img, t) in enumerate(zip(frames, stamps)):
            if k in (2, 3, 11):
                b, g, r = (img[..., c].astype(np.int64) for c in range(3))
                gray = ((b * 3735 + g * 19235 + r * 9798 + 16384) >> 15).astype(np.uint8)
                ps.write_png(str(d / f"{t}.png"), gray)
                decoded.append(np.repeat(gray[:, :, None], 3, 2))
            else:
                ps.write_png(str(d / f"{t}.png"), img)
                decoded.append(img)
        out[name] = dict(dir=d, stamps=stamps, decoded=np.stack(decoded), has_board=np.array(has_board))
    return out


def _cli(folder, out, env=None):
    r = subprocess.run([os.path.join(BIN, "extract_board_to_json"), "--input_path", str(folder), "--board_type", "radon", "--num_squares_x", str(W),
                        "--num_squares_y", str(H), "--checker_square_length_m", str(SQ), "--downsample_factor", str(FACTOR),
                        "--save_corners_json_path", str(out), "--recompute_corners"], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr + r.stdout
    return r


@pytest.fixture(scope="module")
def runs(folders, tmp_path_factory):
    out = {}
    for name, F in folders.items():
        path = tmp_path_factory.mktemp(name + "_out") / "corners.uson"
        r = _cli(F["dir"], path)
        print(r.stdout)
        out[name] = path
    return out


@pytest.mark.parametrize("name", list(CAMERAS))
def test_cli_file_layout_and_corners(api, folders, runs, name):
    F = folders[name]
    data = open(runs[name], "rb").read()
    doc = io_formats.ubjson_loads(data)
    assert sorted(doc) == ["calibration_board_type", "camera_fps", "image_height", "image_width", "scene_pts", "square_size_meter", "views"]
    assert doc["calibration_board_type"] == 1
    s = np.float32(SQ)
    assert doc["square_size_meter"] == float(s)
    assert doc["scene_pts"] == [[float(np.float32(i) * s), float(np.float32(j) * s), 0.0] for i in range(H) for j in range(W)]
    assert (doc["image_width"], doc["image_height"]) == (640, 360)
    t = sorted(set(int(x) * 1e-9 for x in F["stamps"]))
    dts = [t[i + 1] - t[i] for i in range(len(t) - 2)]
    assert doc["camera_fps"] == 1.0 / float(np.median(dts))
    assert doc["camera_fps"] != 1.0 / float(np.median(np.diff(t)))   # the dropped last interval matters for these stamps
    uv, found, _ = api.extract_radon_board_bgr(F["decoded"], W, H, FACTOR)
    np.testing.assert_array_equal(found, F["has_board"])
    keys = [f"{int(x) * 1e-9 * 1e6:f}" for x in F["stamps"]]
    assert sorted(doc["views"]) == sorted(k for k, f in zip(keys, found) if f)
    for k, key in enumerate(keys):
        if found[k]:
            ip = doc["views"][key]["image_points"]
            assert sorted(ip, key=int) == [str(c) for c in range(W * H)]
            np.testing.assert_array_equal(np.array([ip[str(c)] for c in range(W * H)]), uv[k])
    # the same bytes for any chunking of the GPU work
    for chunk in ("1", "7"):
        other = runs[name].parent / f"chunk{chunk}.uson"
        _cli(F["dir"], other, env=dict(os.environ, ICC_BOARD_CHUNK_FRAMES=chunk))
        assert open(other, "rb").read() == data, chunk


@pytest.mark.parametrize("name", list(CAMERAS))
def test_calibrate_camera_on_the_cli_output(runs, name, tmp_path):
    model_name, model, intr, _ = CAMERAS[name]
    out = tmp_path / "calib"
    r = subprocess.run([os.path.join(BIN, "calibrate_camera"), "--input_corners", str(runs[name]), "--camera_model_to_calibrate", model_name,
                        "--save_path_calib_dataset", str(out), "--grid_size=0"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    cal = json.load(open(str(out) + ".json"))
    k = cal["intrinsics"]
    f_true, cx_true, cy_true = intr[0] / FACTOR, (intr[3] + 0.5) / FACTOR - 0.5, (intr[4] + 0.5) / FACTOR - 0.5
    err = (k["focal_length"] - f_true, k["principal_pt_x"] - cx_true, k["principal_pt_y"] - cy_true)
    print(f"{name}: focal length error {err[0]:+.3f} px, principal point error ({err[1]:+.3f}, {err[2]:+.3f}) px, "
          f"{cal['nr_calib_images']} views, reprojection error {cal['final_reproj_error']:.4f} px")
    assert max(abs(e) for e in err) < 1.0, err
    # the Python calibrator reads the array-form scene_pts as well
    cc = calibrator.CameraCalibrator(model_name)
    cc.SetGridSize(0.0)
    assert cc.CalibrateCameraFromJson(io_formats.ubjson_loads(open(runs[name], "rb").read()))
    assert abs(cc.result["intrinsics"][0] - k["focal_length"]) < 1e-6 * k["focal_length"]
