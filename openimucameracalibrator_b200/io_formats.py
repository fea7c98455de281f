"""File formats of the hot CLI (SURVEY.md §8(b)): writers used to turn a synthetic dataset into the exact files that
`continuous_time_imu_to_camera_calibration` reads, and a reader for its result JSON.

  corners      UBJSON  (src/core/board_extractor.cc:294-296,325-333,375-380 -> nlohmann::json::to_ubjson)
  camera       JSON    (src/io/read_camera_calibration.cc:35-119)
  telemetry    JSON    (src/io/read_telemetry.cc:29-69)
  sew          JSON    (src/io/read_misc.cc:30-46)
  init         JSON    (src/io/read_misc.cc:63-82)
  bias         JSON    (src/io/read_misc.cc:48-61)
  imu intr.    JSON    (src/io/read_misc.cc:84-150)
  pose dataset JSON stand-in for Theia's cereal-binary .calibdata (see csrc/continuous_time_imu_to_camera_calibration.cpp)
"""
from __future__ import annotations

import json
import os
import struct

import numpy as np

from . import camera_models as cm


# ---- UBJSON (draft 12), the subset nlohmann::json::to_ubjson emits without size/type optimisation -------------------
def _ub_int(n: int) -> bytes:
    if -128 <= n <= 127:
        return b"i" + struct.pack(">b", n)
    if 0 <= n <= 255:
        return b"U" + struct.pack(">B", n)
    if -32768 <= n <= 32767:
        return b"I" + struct.pack(">h", n)
    if -2 ** 31 <= n < 2 ** 31:
        return b"l" + struct.pack(">i", n)
    return b"L" + struct.pack(">q", n)


def ubjson_dumps(v) -> bytes:
    if v is None:
        return b"Z"
    if isinstance(v, bool):
        return b"T" if v else b"F"
    if isinstance(v, (int, np.integer)):
        return _ub_int(int(v))
    if isinstance(v, (float, np.floating)):
        return b"D" + struct.pack(">d", float(v))
    if isinstance(v, str):
        b = v.encode()
        return b"S" + _ub_int(len(b)) + b
    if isinstance(v, (list, tuple, np.ndarray)):
        return b"[" + b"".join(ubjson_dumps(x) for x in v) + b"]"
    if isinstance(v, dict):
        out = [b"{"]
        for k in sorted(v):            # nlohmann's object is a std::map: keys are emitted sorted
            kb = str(k).encode()
            out.append(_ub_int(len(kb)) + kb + ubjson_dumps(v[k]))
        out.append(b"}")
        return b"".join(out)
    raise TypeError(type(v))


def ubjson_loads(data: bytes):
    pos = 0

    def integer(t):
        nonlocal pos
        fmt = {"i": ">b", "U": ">B", "I": ">h", "l": ">i", "L": ">q"}[t]
        n = struct.calcsize(fmt); val = struct.unpack_from(fmt, data, pos)[0]; pos += n
        return val

    def raw_string():
        nonlocal pos
        t = chr(data[pos]); pos += 1
        n = integer(t); s = data[pos:pos + n].decode(); pos += n
        return s

    def value():
        nonlocal pos
        t = chr(data[pos]); pos += 1
        if t == "Z":
            return None
        if t in "TF":
            return t == "T"
        if t in "iUIlL":
            return integer(t)
        if t == "d":
            v = struct.unpack_from(">f", data, pos)[0]; pos += 4; return v
        if t == "D":
            v = struct.unpack_from(">d", data, pos)[0]; pos += 8; return v
        if t == "S":
            return raw_string()
        if t == "[":
            out = []
            while chr(data[pos]) != "]":
                out.append(value())
            pos += 1
            return out
        if t == "{":
            out = {}
            while chr(data[pos]) != "}":
                k = raw_string(); out[k] = value()
            pos += 1
            return out
        raise ValueError(f"ubjson: unknown marker {t!r} at {pos}")
    return value()


# ---- dataset -> files -----------------------------------------------------------------------------------------------------
def intrinsics_dict(model: int, k) -> dict:
    """The `intrinsics` object of the camera JSON for Theia-ordered intrinsics k: every key of the model's layout, and `skew` 0.0 for
    the models whose index 2 is no skew (the readers never read `skew`)."""
    intr = {key: float(k[i]) for key, i in cm.CAMERAS[model].keys.items()}
    intr.setdefault("skew", 0.0)
    return intr


def view_key(t_s: float) -> str:
    """BoardExtractor stores views under std::to_string(double timestamp_us) (six decimals)."""
    return f"{t_s * 1e6:.6f}"


def write_dataset_files(ds: dict, out_dir: str) -> dict:
    """Write every input file of the hot CLI for a synthetic dataset; returns {flag name: path}."""
    os.makedirs(out_dir, exist_ok=True)
    W, H = ds["image_size"]
    paths = {}
    # corners (UBJSON)
    off, ids, uv = ds["corner_offsets"], ds["point_ids"], ds["uv"]
    views = {}
    for f, t in enumerate(ds["frame_t"]):
        views[view_key(float(t))] = {"image_points": {str(int(ids[c])): [float(uv[c, 0]), float(uv[c, 1])] for c in range(off[f], off[f + 1])}}
    scene = {"calibration_board_type": "charuco", "square_size_meter": 0.021, "camera_fps": float(ds["fps"]), "image_width": int(W), "image_height": int(H),
             "scene_pts": {str(i): [float(p[0]), float(p[1]), float(p[2])] for i, p in enumerate(ds["board_xyzw"])}, "views": views}
    paths["input_corners"] = os.path.join(out_dir, "corners.uson")
    with open(paths["input_corners"], "wb") as f:
        f.write(ubjson_dumps(scene))
    # camera calibration
    cam = {"fps": float(ds["fps"]), "image_width": int(W), "image_height": int(H), "intrinsic_type": cm.MODEL_NAMES[ds["model"]], "intrinsics": intrinsics_dict(ds["model"], ds["intrinsics"])}
    paths["camera_calibration_json"] = os.path.join(out_dir, "cam_calib.json")
    json.dump(cam, open(paths["camera_calibration_json"], "w"), indent=4)
    # telemetry (timestamps as integer nanoseconds like telemetry_converter.py)
    tel = {"timestamps_ns": [int(round(t * 1e9)) for t in ds["imu_t"]], "accelerometer": np.asarray(ds["accel"]).tolist(), "gyroscope": np.asarray(ds["gyro"]).tolist(),
           "img_timestamps_ns": []}
    paths["telemetry_json"] = os.path.join(out_dir, "telemetry.json")
    json.dump(tel, open(paths["telemetry_json"], "w"))
    # spline error weighting
    sew = {"camera_fps": float(ds["fps"]), "r3": {"knot_spacing": ds["dt_r3_s"], "weighting_factor": ds["std_r3"]}, "so3": {"knot_spacing": ds["dt_so3_s"], "weighting_factor": ds["std_so3"]}}
    paths["spline_error_weighting_json"] = os.path.join(out_dir, "sew.json")
    json.dump(sew, open(paths["spline_error_weighting_json"], "w"), indent=4)
    # gyro -> camera initialisation: the file stores q_gyro_to_cam = q_i_c^-1  (app :170 conjugates it back)
    q = ds["T_i_c_init"][:4]
    init = {"gyro_to_camera_rotation": {"w": float(q[3]), "x": float(-q[0]), "y": float(-q[1]), "z": float(-q[2])}, "time_offset_gyro_to_cam": float(ds["time_offset_imu_to_cam_s"])}
    paths["gyro_to_cam_initial_calibration"] = os.path.join(out_dir, "imu_to_cam_init.json")
    json.dump(init, open(paths["gyro_to_cam_initial_calibration"], "w"), indent=4)
    # biases
    b = {"accl_bias": dict(zip("xyz", map(float, ds["acc_bias"]))), "gyro_bias": dict(zip("xyz", map(float, ds["gyr_bias"])))}
    paths["imu_bias_file"] = os.path.join(out_dir, "imu_bias.json")
    json.dump(b, open(paths["imu_bias_file"], "w"), indent=4)
    # pose dataset (JSON stand-in for .calibdata); view name = to_string((uint64) timestamp_us)
    pv = {}
    for f, t in enumerate(ds["frame_t"]):
        qq = ds["q_wc"][f]
        pv[str(int(float(view_key(float(t)))))] = {"q_wc": [float(qq[3]), float(qq[0]), float(qq[1]), float(qq[2])], "p_wc": [float(x) for x in ds["p_wc"][f]]}
    pose = {"views": pv, "tracks": {str(i): [float(x) for x in p] for i, p in enumerate(ds["board_xyzw"])}}
    paths["input_pose_dataset"] = os.path.join(out_dir, "pose_dataset.json")
    json.dump(pose, open(paths["input_pose_dataset"], "w"))
    return paths


def dataset_from_files(ds: dict) -> dict:
    """What the CLI sees after the files' rounding: view timestamps go through `%f` microseconds, IMU stamps through int ns."""
    d = dict(ds)
    d["frame_t"] = np.array([float(view_key(float(t))) * 1e-6 for t in ds["frame_t"]])
    d["imu_t"] = np.array([int(round(t * 1e9)) * 1e-9 for t in ds["imu_t"]])
    order = np.argsort([view_key(float(t)) for t in ds["frame_t"]], kind="stable")     # std::map iteration order of the view keys
    off = np.asarray(ds["corner_offsets"])
    new_off, ids, uv = [0], [], []
    for f in order:
        # image_points is a std::map<string,...> too: ids are visited in lexicographic order of their decimal strings
        cs = sorted(range(off[f], off[f + 1]), key=lambda c: str(int(ds["point_ids"][c])))
        ids += [ds["point_ids"][c] for c in cs]; uv += [ds["uv"][c] for c in cs]; new_off.append(len(ids))
    d["corner_offsets"] = np.array(new_off, dtype=np.int32); d["point_ids"] = np.array(ids, dtype=np.int32); d["uv"] = np.array(uv).reshape(-1, 2)
    d["frame_t"] = d["frame_t"][order]; d["q_wc"] = np.asarray(ds["q_wc"])[order]; d["p_wc"] = np.asarray(ds["p_wc"])[order]
    return d


def read_result_json(path: str) -> dict:
    return json.load(open(path))


def imu_intrinsics_document(acc_params, gyr_params, gyr_bias) -> dict:
    """The IMU intrinsics JSON of applications/static_imu_calibration.cc:60-85 (read by the hot CLI's --imu_intrinsics): accelerometer
    misalignment upper triangular with a unit diagonal, gyroscope misalignment full, diagonal scale matrices, 3-vector biases.
    acc_params [misYZ, misZY, misZX, sX, sY, sZ, bX, bY, bZ]; gyr_params [misYZ, misZY, misZX, misXZ, misXY, misYX, sX, sY, sZ]."""
    a = [float(v) for v in acc_params]; g = [float(v) for v in gyr_params]
    return {
        "accelerometer": {"misalignment_matrix": [[1.0, -a[0], a[1]], [0.0, 1.0, -a[2]], [0.0, 0.0, 1.0]],
                          "scale_matrix": [[a[3], 0.0, 0.0], [0.0, a[4], 0.0], [0.0, 0.0, a[5]]], "bias": a[6:9]},
        "gyroscope": {"misalignment_matrix": [[1.0, -g[0], g[1]], [g[3], 1.0, -g[2]], [-g[4], g[5], 1.0]],
                      "scale_matrix": [[g[6], 0.0, 0.0], [0.0, g[7], 0.0], [0.0, 0.0, g[8]]], "bias": [float(v) for v in gyr_bias]},
    }


def write_imu_intrinsics_json(path: str, acc_params, gyr_params, gyr_bias) -> None:
    with open(path, "w") as f:
        json.dump(imu_intrinsics_document(acc_params, gyr_params, gyr_bias), f, indent=4)


def allan_variance_document(result: dict, curves: list) -> dict:
    """The --output_json document of bin/fit_allan_variance: per channel (acc_x .. gyr_z) the curve (factors, tau [s], sigma2, fitted
    deviation), the fitted [Q, N, B, K, R], the derived noise quantities and the fit statistics.  `result` is CApi.allan_variance's,
    `curves` the six CApi.allan_curves dicts."""
    from ._capi import ALLAN_CHANNELS, ALLAN_PARAMS
    s0 = result["summary"][0]
    doc = {"n_samples": float(s0["n_samples"]), "freq": float(s0["freq"]), "period": float(s0["period"]), "channels": {}}
    for c, name in enumerate(ALLAN_CHANNELS):
        cv, s = curves[c], result["summary"][c]
        doc["channels"][name] = {
            "factors": [float(v) for v in cv["factors"]], "tau": [float(v) for v in cv["tau"]], "sigma2": [float(v) for v in cv["sigma2"]],
            "fit_deviation": [float(v) for v in cv["fit_deviation"]],
            "params": {k: float(v) for k, v in zip(ALLAN_PARAMS, result["params"][c])},
            "noise": {k: float(v) for k, v in result["noise"][c].items()},
            "fit": {"points": float(s["n_fit_points"]), "iterations": float(s["iterations"]), "termination": float(s["termination"]),
                    "initial_cost": float(s["initial_cost"]), "final_cost": float(s["final_cost"])},
        }
    return doc


# Allan-deviation scale of each sensor's fit: the accelerometer in m/s^2, the gyroscope in deg/h (57.3 deg/rad, 3600 s/h)
ALLAN_RATE_SCALE = {"acc": 1.0, "gyr": 57.3 * 3600}


def bias_random_walk_from_allan(doc: dict):
    """(acc_q[3], gyr_q[3]) random-walk densities in Kalibr's units (m/s^3/sqrt(Hz), rad/s^2/sqrt(Hz)) from a fit_allan_variance
    --output_json document: per axis q = sqrt(3) |K| / scale, K the fitted rate-random-walk term of that channel's Allan variance."""
    ch = doc["channels"]
    q = {s: np.array([np.sqrt(3.0) * abs(float(ch[f"{s}_{a}"]["params"]["K"])) / ALLAN_RATE_SCALE[s] for a in "xyz"]) for s in ("acc", "gyr")}
    return q["acc"], q["gyr"]


def write_allan_variance_json(path: str, result: dict, curves: list) -> None:
    with open(path, "w") as f:
        json.dump(allan_variance_document(result, curves), f, indent=1)
