"""Golden vectors for the static IMU bias step, produced by the REFERENCE'S OWN code: python/get_imu_biases.py of
urbste/OpenImuCameraCalibrator is plain NumPy, so its unmodified main() is run here (from a checkout of the reference named by
$ICC_REFERENCE_ROOT) on deterministic telemetry files and inputs + outputs are committed as tests/golden/imu_bias_*.npz.

The script imports matplotlib (plots that are commented out) and the container has none: an empty stand-in module is registered for
the import to succeed -- no line of the reference is changed or skipped.
Run from the repo root:  ICC_REFERENCE_ROOT=<reference checkout> python tests/golden/make_imu_bias_golden.py
"""
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np

REF_PY = os.path.join(os.environ["ICC_REFERENCE_ROOT"], "python")
OUT = os.path.dirname(os.path.abspath(__file__))


def run_reference(telemetry: dict, gravity_const: float, remove_sec: float) -> dict:
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, REF_PY)
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "telemetry.json"), os.path.join(d, "bias.json")
        json.dump(telemetry, open(src, "w"))
        argv = sys.argv
        sys.argv = ["get_imu_biases.py", "--input_json_path", src, "--output_path", dst, "--gravity_const", repr(gravity_const), "--remove_sec", repr(remove_sec)]
        try:
            runpy.run_path(os.path.join(REF_PY, "get_imu_biases.py"), run_name="__main__")
        finally:
            sys.argv = argv
        return json.load(open(dst))


def stream(n, rate, seed, axis, sign):
    rng = np.random.default_rng(seed)
    t = (np.arange(n) / rate * 1e9).astype(np.int64)
    g = np.zeros(3); g[axis] = sign * 9.8065
    accl = g + np.array([0.05, -0.03, 0.02]) + rng.normal(0, 0.06, (n, 3)) + 0.2 * np.sin(np.arange(n)[:, None] / rate * np.array([1.3, 0.7, 2.1]))
    gyro = np.array([2e-3, -1e-3, 5e-4]) + rng.normal(0, 4e-3, (n, 3))
    return {"accelerometer": accl.tolist(), "gyroscope": gyro.tolist(), "timestamps_ns": t.tolist(), "img_timestamps_ns": [], "camera_fps": 30.0}


def main():
    cases = [("z_up_200hz", stream(4001, 200.0, 1, 2, +1), 9.81, 0.0), ("y_down_trimmed", stream(6000, 400.0, 2, 1, -1), 9.80665, 1.5),
             ("x_up_1khz", stream(8000, 1000.0, 3, 0, +1), 9.811104, 0.25)]
    for name, tel, gc, rs in cases:
        out = run_reference(tel, gc, rs)
        np.savez_compressed(os.path.join(OUT, f"imu_bias_{name}.npz"), accelerometer=np.array(tel["accelerometer"]), gyroscope=np.array(tel["gyroscope"]),
                            timestamps_ns=np.array(tel["timestamps_ns"]), gravity_const=gc, remove_sec=rs,
                            accl_bias=np.array([out["accl_bias"][k] for k in "xyz"]), gyro_bias=np.array([out["gyro_bias"][k] for k in "xyz"]))
        print(name, out)


if __name__ == "__main__":
    main()
