"""Drop-in for python/get_sew_for_dataset.py of urbste/OpenImuCameraCalibrator (SURVEY.md §8(f) row f2): same command line
(--input_json_path, --output_path, --q_so3, --q_r3), same telemetry JSON in (accelerometer, gyroscope, timestamps_ns, camera_fps),
same spline_error_weighting JSON out ({"so3": {knot_spacing, weighting_factor, quality_factor}, "r3": {...}, "camera_fps"}), which is
what the hot CLI reads as --spline_error_weighting_json.  The spectra and the knot-spacing searches run on the GPU through
icc_spline_error_weighting (python/sew.py:knot_spacing_and_variance); there is no CPU fallback.

    python -m openimucameracalibrator_b200.get_sew_for_dataset --input_json_path telemetry.json --output_path sew.json
"""
from __future__ import annotations

import json
from argparse import ArgumentParser

import numpy as np

from . import _capi as capi
from .calibrator import load_library


def spline_error_weighting(telemetry: dict, q_so3: float = 0.98, q_r3: float = 0.96, device: int = 0) -> dict:
    """python/get_sew_for_dataset.py:34-62 on an already parsed telemetry dictionary."""
    accl = np.asarray(telemetry["accelerometer"], dtype=np.float64)
    gyro = np.asarray(telemetry["gyroscope"], dtype=np.float64)
    t = np.asarray(telemetry["timestamps_ns"], dtype=np.float64).squeeze() * 1e-9
    api = capi.CApi(load_library(), "icc_", device)
    r3_dt, r3_var = api.spline_error_weighting(t, accl, q_r3, 0.01, 0.15)        # :38
    so3_dt, so3_var = api.spline_error_weighting(t, gyro, q_so3, 0.01, 0.2)      # :39
    fps = float(telemetry.get("camera_fps", 0.0) or 0.0)
    return {"so3": {"knot_spacing": so3_dt, "weighting_factor": float(np.sqrt(so3_var)), "quality_factor": q_so3},
            "r3": {"knot_spacing": r3_dt, "weighting_factor": float(np.sqrt(r3_var)), "quality_factor": q_r3},
            "camera_fps": fps if fps != 0.0 else 30.0}


def main(argv=None):
    parser = ArgumentParser()
    parser.add_argument("--input_json_path", default="", help="path to metadata json")
    parser.add_argument("--output_path", help="output path")
    parser.add_argument("--q_so3", help="quality value for rotational component, i.e. gyro signal", default=0.98, type=float)
    parser.add_argument("--q_r3", help="quality value for translational component, i.e. accelerometer signal", default=0.96, type=float)
    parser.add_argument("--use_gopro_importer", default=0, help="accepted for compatibility; only the generic telemetry JSON is read")
    parser.add_argument("--device", default=0, type=int, help="CUDA ordinal (extra flag)")
    args = parser.parse_args(argv)
    with open(args.input_json_path) as f:
        telemetry = json.load(f)
    sew = spline_error_weighting(telemetry, args.q_so3, args.q_r3, args.device)
    print("Knot spacing SO3:               {:.3f} seconds at quality level q_so3={}".format(sew["so3"]["knot_spacing"], args.q_so3))
    print("Knot spacing  R3:               {:.3f} seconds at quality level q_r3={}".format(sew["r3"]["knot_spacing"], args.q_r3))
    print("Gyroscope weighting factor:     {:.3f} at quality level q_so3={}".format(1.0 / sew["so3"]["weighting_factor"], args.q_so3))
    print("Accelerometer weighting factor: {:.3f} at quality level q_r3={}".format(1.0 / sew["r3"]["weighting_factor"], args.q_r3))
    print("Writing result to: ", args.output_path)
    with open(args.output_path, "w") as f:
        json.dump(sew, f)
    return sew


if __name__ == "__main__":
    main()
