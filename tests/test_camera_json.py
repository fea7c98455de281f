"""The camera JSON and the printed camera summary, for every camera model, on the CPU: the layout stated here once by hand against the
Python table (camera_models.CAMERAS); the Python writer (io_formats.intrinsics_dict) read back by the hot CLI (`--parse_only`); the C++
writer (icc_cli_common.hpp, through tests/camera_json/camera_json_shim.cpp) against the Python writer and read back the same way; the C++
printer against CameraCalibrator.PrintResult; FOV's optional aspect ratio and the reader's error messages."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import calibrator
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")

_AFFINE = {"focal_length": 0, "aspect_ratio": 1, "skew": 2, "principal_pt_x": 3, "principal_pt_y": 4}
# intrinsic_type -> (parameter count, JSON key -> Theia index); `skew` is listed where index 2 is the skew
LAYOUT = {
    "PINHOLE": (7, dict(_AFFINE)),
    "PINHOLE_RADIAL_TANGENTIAL": (10, dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, tangential_distortion_1=8,
                                           tangential_distortion_2=9)),
    "FISHEYE": (9, dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, radial_distortion_4=8)),
    "FOV": (5, dict(focal_length=0, aspect_ratio=1, principal_pt_x=2, principal_pt_y=3, radial_distortion_1=4)),
    "DIVISION_UNDISTORTION": (5, dict(focal_length=0, aspect_ratio=1, principal_pt_x=2, principal_pt_y=3, div_undist_distortion=4)),
    "DOUBLE_SPHERE": (7, dict(_AFFINE, xi=5, alpha=6)),
    "EXTENDED_UNIFIED": (7, dict(_AFFINE, alpha=5, beta=6)),
    "OMNI_RADIAL_TANGENTIAL": (10, dict(_AFFINE, xi=5, radial_distortion_1=6, radial_distortion_2=7, tangential_distortion_1=8, tangential_distortion_2=9)),
    "SCARAMUZZA": (9, dict(focal_length=0, aspect_ratio=1, stretch_e=2, principal_pt_x=3, principal_pt_y=4, polynomial_a2=5, polynomial_a3=6,
                           polynomial_a4=7, stretch_d=8)),
    "PINHOLE_RATIONAL": (13, dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, tangential_distortion_1=8,
                                  tangential_distortion_2=9, radial_distortion_4=10, radial_distortion_5=11, radial_distortion_6=12)),
}
# the model line of PrintResult, str.format of the intrinsics; None: no line
PRINTED = {
    "PINHOLE": None, "PINHOLE_RADIAL_TANGENTIAL": None, "FOV": None,
    "FISHEYE": "FISHEYE model: Radial distortion 1: {5} Radial distortion 2: {6} Radial distortion 3: {7} Radial distortion 4: {8}",
    "DIVISION_UNDISTORTION": "DIVISION_UNDISTORTION model: Distortion: {4}",
    "DOUBLE_SPHERE": "DOUBLE_SPHERE model: XI: {5} ALPHA: {6}",
    "EXTENDED_UNIFIED": "EXTENDED_UNIFIED model: {5} BETA: {6}",
    "OMNI_RADIAL_TANGENTIAL": "OMNI_RADIAL_TANGENTIAL model: XI: {5} Radial distortion 1: {6} Radial distortion 2: {7} Tangential distortion 1: {8} "
                              "Tangential distortion 2: {9}",
    "SCARAMUZZA": "SCARAMUZZA model: A2: {5} A3: {6} A4: {7} Stretch c: {1} d: {8} e: {2}",
    "PINHOLE_RATIONAL": "PINHOLE_RATIONAL model: Radial distortion 1: {5} Radial distortion 2: {6} Radial distortion 3: {7} Radial distortion 4: {10} "
                        "Radial distortion 5: {11} Radial distortion 6: {12} Tangential distortion 1: {8} Tangential distortion 2: {9}",
}
NAMES = list(LAYOUT)


def _k(name):
    """seeded intrinsics without a short decimal form, every index (the skew too) non-zero and distinct"""
    n = LAYOUT[name][0]
    return np.random.default_rng(n + len(name)).uniform(0.5, 2.0, n) * np.array([1e3, 1.0, 1e-2, 1e3, 1e3] + [0.1] * (n - 5))


@pytest.fixture(scope="module")
def base_ds():
    return syn.make_dataset(syn.tiny_config(n_frames=4))


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("camera_json") / "camera_json_shim")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-o", out, os.path.join(HERE, "camera_json", "camera_json_shim.cpp")])
    return lambda *a: subprocess.run([out, *a], capture_output=True, text=True)


def _files(base_ds, name, k, tmp_path):
    return iof.write_dataset_files(dict(base_ds, model=cm.MODEL_IDS[name], intrinsics=k), str(tmp_path))


def _parse_only(paths, tmp_path):
    assert os.path.exists(HOT_CLI), "build the CLI first (__graft_entry__.build())"
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/result.json", f"--output_path={tmp_path}", "--parse_only"]
    return subprocess.run(args, capture_output=True, text=True)


def _read_back(name, k):
    """what the readers give back: every carried index but the skew, which is never read; 0 elsewhere (PINHOLE's k5, k6)"""
    out = np.zeros(LAYOUT[name][0])
    for key, i in LAYOUT[name][1].items():
        out[i] = 0.0 if key == "skew" else k[i]
    return out


@pytest.mark.parametrize("name", NAMES)
def test_layout_is_the_python_table(name):
    n, keys = LAYOUT[name]
    c = cm.CAMERAS[cm.MODEL_IDS[name]]
    assert c.name == cm.MODEL_NAMES[c.id] == name and c.num_params == cm.NUM_PARAMS[c.id] == n
    assert c.keys == keys
    if name == "PINHOLE":
        assert sorted(keys.values()) == [0, 1, 2, 3, 4]
    else:
        assert sorted(keys.values()) == list(range(n))                # every other model carries every index


@pytest.mark.parametrize("name", NAMES)
def test_python_writer_to_cli_reader(name, base_ds, tmp_path):
    k = _k(name)
    paths = _files(base_ds, name, k, tmp_path)
    cam = json.load(open(paths["camera_calibration_json"]))
    expected = {key: float(k[i]) for key, i in LAYOUT[name][1].items()}
    expected.setdefault("skew", 0.0)
    assert cam["intrinsic_type"] == name and cam["intrinsics"] == expected
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    s = json.loads(out.stdout)
    assert s["camera_model"] == cm.MODEL_IDS[name] and np.array_equal(np.array(s["intrinsics"]), _read_back(name, k))
    # every key the reader reads is required, except FOV's aspect ratio (test_fov_aspect_ratio_is_optional)
    for key in LAYOUT[name][1]:
        if key == "skew" or (name == "FOV" and key == "aspect_ratio"):
            continue
        doc = json.loads(json.dumps(cam))
        del doc["intrinsics"][key]
        json.dump(doc, open(paths["camera_calibration_json"], "w"))
        out = _parse_only(paths, tmp_path)
        assert out.returncode != 0 and f"missing key '{key}'" in out.stderr, (key, out.stderr)


@pytest.mark.parametrize("name", NAMES)
def test_cpp_writer_against_python_writer_and_reader(name, base_ds, shim, tmp_path):
    k = _k(name)
    out = shim("write", name, *map(repr, map(float, k)))
    assert out.returncode == 0, out.stderr
    written = json.loads(out.stdout)
    assert written == iof.intrinsics_dict(cm.MODEL_IDS[name], k)
    paths = _files(base_ds, name, k, tmp_path)
    cam = json.load(open(paths["camera_calibration_json"]))
    cam["intrinsics"] = written
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    assert np.array_equal(np.array(json.loads(out.stdout)["intrinsics"]), _read_back(name, k))


_PY_FLOAT = re.compile(r"-?\d+\.\d+(?:e[-+]\d+)?|-?\d+e[-+]\d+")


@pytest.mark.parametrize("name", NAMES)
def test_cpp_printer_against_python_printer(name, shim, monkeypatch, capsys):
    k = _k(name)
    monkeypatch.setattr(calibrator, "load_library", lambda: None)
    monkeypatch.setattr(calibrator, "CApi", lambda *a: None)
    cal = calibrator.CameraCalibrator(name)
    cal.result = {"intrinsics": k}
    cal.PrintResult()
    py = capsys.readouterr().out
    pp = LAYOUT[name][1]
    lines = [f"Focal Length:{k[0]}px Principal Point: {k[pp['principal_pt_x']]}/{k[pp['principal_pt_y']]}px."]
    if PRINTED[name]:
        lines.append(PRINTED[name].format(*k))
    assert py == "".join(line + "\n" for line in lines)
    out = shim("print", name, *map(repr, map(float, k)))
    assert out.returncode == 0, out.stderr
    # the same labels, and the numbers as std::ostream prints them: six significant digits
    assert out.stdout == _PY_FLOAT.sub(lambda m: format(float(m.group()), "g"), py)


def test_fov_aspect_ratio_is_optional(base_ds, tmp_path):
    k = _k("FOV")
    paths = _files(base_ds, "FOV", k, tmp_path)
    cam = json.load(open(paths["camera_calibration_json"]))
    del cam["intrinsics"]["aspect_ratio"]
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode == 0, out.stderr
    expected = k.copy(); expected[1] = 1.0
    assert np.array_equal(np.array(json.loads(out.stdout)["intrinsics"]), expected)


def test_unknown_intrinsic_type(base_ds, tmp_path):
    paths = _files(base_ds, "PINHOLE", _k("PINHOLE"), tmp_path)
    cam = json.load(open(paths["camera_calibration_json"]))
    cam["intrinsic_type"] = "NO_SUCH_MODEL"
    json.dump(cam, open(paths["camera_calibration_json"], "w"))
    out = _parse_only(paths, tmp_path)
    assert out.returncode != 0 and "unknown intrinsic_type NO_SUCH_MODEL" in out.stderr
