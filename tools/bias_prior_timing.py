"""Time the LM iteration of BASELINE config 4 (3000 views x 144 corners, EXTENDED_UNIFIED, 100 s) on one GPU with the biases free
(SPLINE | T_I_C | IMU_BIASES) in three settings: the reference's 10 s bias splines without a prior, 2 s bias splines without a prior, and
2 s bias splines with the random-walk prior (icc_set_bias_random_walk).  Each setting runs `--iters` LM iterations (icc_lm_iterations: no
convergence test, one Jacobian evaluation per accepted step) `--repeats` times after a warm-up; the time is the host clock around the call,
which ends with a stream synchronisation.  Also times the prior kernel alone through icc_time_evaluations (Jacobian mode) as the
difference of the two 2 s settings.  Prints one JSON line.
usage: python tools/bias_prior_timing.py [--iters N] [--repeats N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn  # noqa: E402

F_BIAS = capi.FLAG_SPLINE | capi.FLAG_T_I_C | capi.FLAG_IMU_BIASES


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    ds = syn.make_dataset(syn.CONFIGS[4])
    lib = calibrator.load_library()
    res = {"gpu": gpu_name(), "iters": a.iters, "repeats": a.repeats}
    settings = {"10s_no_prior": (10.0, (None, None)), "2s_no_prior": (2.0, (None, None)), "2s_prior": (2.0, (2e-3, 2e-4))}
    for name, (dt, walk) in settings.items():
        per_iter, eval_ms = [], []
        g = capi.CApi(lib, "icc_", 0)
        g.set_bias_splines(dt, dt); g.set_bias_random_walk(*walk)
        capi.load_dataset(g, ds)
        so3, r3, ba, bg = g.get_knots(); T = g.get_T_i_c()
        for r in range(a.repeats + 1):                 # round 0 warms every kernel up and is not reported
            g.set_knots(so3, r3, ba, bg); g.set_T_i_c(T)
            t0 = time.perf_counter(); s = g.lm_iterations(a.iters, F_BIAS); t1 = time.perf_counter()
            if r:
                per_iter.append((t1 - t0) * 1e3 / max(1, s.iterations))
                eval_ms.append(g.time_evaluations(20, F_BIAS, with_jacobian=True))
        res[name] = dict(lm_ms_per_iteration_median=float(np.median(per_iter)), lm_ms_per_iteration_range=[min(per_iter), max(per_iter)],
                         jacobian_eval_ms_median=float(np.median(eval_ms)), prior_rows=g.num_bias_prior_residuals(), bias_knots=g.num_knots()[2],
                         border_columns=g.num_tangent(F_BIAS) - 3 * (g.num_knots()[0] + g.num_knots()[1]))
        g.close()
    res["prior_overhead_ms_per_iteration"] = res["2s_prior"]["lm_ms_per_iteration_median"] - res["2s_no_prior"]["lm_ms_per_iteration_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
