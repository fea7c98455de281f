"""Drop-in for python/get_imu_biases.py of urbste/OpenImuCameraCalibrator: same command line (--input_json_path, --output_path,
--gravity_const, --remove_sec), same telemetry JSON in, same bias JSON out ({"gyro_bias": {x,y,z}, "accl_bias": {x,y,z}}), which is what
the hot CLI reads as --imu_bias_file and estimate_imu_to_camera_rotation as --imu_bias_estimate.  The stream reductions run on the GPU
through icc_estimate_imu_biases; there is no CPU fallback.

    python -m openimucameracalibrator_b200.get_imu_biases --input_json_path telemetry.json --output_path imu_bias.json
"""
from __future__ import annotations

import json
from argparse import ArgumentParser

import numpy as np

from . import _capi as capi
from .calibrator import load_library


def remove_seconds(accl, gyro, timestamps_ns, skip_seconds):
    """TelemetryImporter._remove_seconds + the truncation of read_generic_json (python/telemetry_converter.py:18-29, 228-232)."""
    if skip_seconds != 0.0:
        nr_remove = round((skip_seconds / 1e-9) / (timestamps_ns[1] - timestamps_ns[0]))
        n = len(timestamps_ns)
        accl, gyro, timestamps_ns = accl[nr_remove:n - nr_remove], gyro[nr_remove:n - nr_remove], timestamps_ns[nr_remove:n - nr_remove]
    return accl[0:len(timestamps_ns)], gyro[0:len(timestamps_ns)], timestamps_ns


def imu_biases(telemetry: dict, gravity_const: float = 9.81, remove_sec: float = 0.0, device: int = 0) -> dict:
    """python/get_imu_biases.py:30-57 on an already parsed telemetry dictionary."""
    accl, gyro, _ = remove_seconds(list(telemetry["accelerometer"]), list(telemetry["gyroscope"]), list(telemetry["timestamps_ns"]), remove_sec)
    api = capi.CApi(load_library(), "icc_", device)
    ba, bg = api.estimate_imu_biases(np.asarray(accl, dtype=np.float64), np.asarray(gyro, dtype=np.float64), gravity_const)
    return {"gyro_bias": {"x": float(bg[0]), "y": float(bg[1]), "z": float(bg[2])}, "accl_bias": {"x": float(ba[0]), "y": float(ba[1]), "z": float(ba[2])}}


def main(argv=None):
    parser = ArgumentParser()
    parser.add_argument("--input_json_path", default="", help="path to metadata json")
    parser.add_argument("--output_path", help="output path")
    parser.add_argument("--gravity_const", help="gravity constant", default=9.81, type=float)
    parser.add_argument("--remove_sec", help="How many seconds to remove from start and end of sequence", default=0.0, type=float)
    parser.add_argument("--use_gopro_importer", default=0, help="accepted for compatibility; only the generic telemetry JSON is read")
    parser.add_argument("--device", default=0, type=int, help="CUDA ordinal (extra flag)")
    args = parser.parse_args(argv)
    with open(args.input_json_path) as f:
        telemetry = json.load(f)
    biases = imu_biases(telemetry, args.gravity_const, args.remove_sec, args.device)
    bg, ba = biases["gyro_bias"], biases["accl_bias"]
    print("Estimated biases:")
    print("gyroscope bias:     {:.5f} rad/s, {:.5f} rad/s, {:.5f} rad/s".format(bg["x"], bg["y"], bg["z"]))
    print("accelerometer bias: {:.5f} m/s2,  {:.5f} m/s2,  {:.5f} m/s2".format(ba["x"], ba["y"], ba["z"]))
    print("Writing result to: ", args.output_path)
    with open(args.output_path, "w") as f:
        json.dump(biases, f)
    return biases


if __name__ == "__main__":
    main()
