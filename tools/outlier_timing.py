"""Time the outlier-corner rejection at BASELINE config 4 (3000 views x 144 corners, EXTENDED_UNIFIED) on one GPU: the per-corner error
pass (icc_get_corner_errors), one rejection (error pass, sums, compaction and schedule rebuild: icc_reject_outlier_corners) and the stage-1
re-solve that follows it.  1 % of the corners are displaced by 20-60 px.  Every timed call ends with a stream synchronisation, so the host
clock measures device work.  Prints one JSON line.
usage: python tools/outlier_timing.py [--repeats N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn  # noqa: E402
from outlier_support import inject_outliers  # noqa: E402

F_STAGE1 = capi.FLAG_SPLINE | capi.FLAG_T_I_C


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    ds, idx = inject_outliers(syn.make_dataset(syn.CONFIGS[4]))
    lib = calibrator.load_library()
    res = {"gpu": gpu_name(), "corners": int(len(ds["point_ids"])), "injected": int(len(idx))}
    err_ms, rej_ms, solve_s, iters = [], [], [], []
    for r in range(a.repeats + 1):                  # the first round warms every kernel up and is not reported
        g = capi.CApi(lib, "icc_", 0); capi.load_dataset(g, ds)
        g.optimize(50, F_STAGE1)
        n = int(np.count_nonzero(g.corner_status() == 1)); e = np.zeros(n)
        t0 = time.perf_counter(); g._call("get_corner_errors", [capi.C.c_int, capi.c_double_p], n, capi._dp(e)); t1 = time.perf_counter()
        s = g.reject_outlier_corners(3.0, 1.0); t2 = time.perf_counter()
        S = g.optimize(50, F_STAGE1); t3 = time.perf_counter()
        if r:
            err_ms.append((t1 - t0) * 1e3); rej_ms.append((t2 - t1) * 1e3); solve_s.append(t3 - t2); iters.append(S.iterations)
        res.update(rejected=int(s["n_rejected"]), threshold_px=s["threshold_px"], injected_rejected=bool(np.all(g.corner_status()[idx] == 0)),
                   n_errors=int(e.size))
        g.close()
    med = lambda v: float(np.median(v))  # noqa: E731
    res.update(error_pass_ms_median=med(err_ms), error_pass_ms_range=[min(err_ms), max(err_ms)], reject_ms_median=med(rej_ms),
               reject_ms_range=[min(rej_ms), max(rej_ms)], resolve_s_median=med(solve_s), resolve_iterations=iters, repeats=a.repeats)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
