"""Pixel against tangent reprojection error on BASELINE config 4 (3000 views x 144 corners, ExtendedUnified): the Jacobian evaluation
(icc_time_evaluations: device events around n evaluations) and one LM iteration (host clock around icc_lm_iterations, which ends in a
device synchronise), in alternating runs of the two modes on fresh handles.  Prints the card and its power limit with the numbers.
usage: python tools/tangent_timing.py [--rounds 4] [--evals 20] [--iters 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn  # noqa: E402

F = capi.FLAG_SPLINE | capi.FLAG_T_I_C


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--evals", type=int, default=20)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    ds = syn.make_dataset(syn.CONFIGS[4])
    lib = calibrator.load_library()
    res = {"pixel": {"jac_ms": [], "lm_ms": []}, "tangent": {"jac_ms": [], "lm_ms": []}}
    for r in range(a.rounds):
        for mode in (("pixel", "tangent") if r % 2 == 0 else ("tangent", "pixel")):
            g = capi.CApi(lib, "icc_", 0)
            g.set_reprojection_error(mode)
            capi.load_dataset(g, ds)
            g.time_evaluations(3, F, True)                                  # warm-up: modules, allocations, layout
            res[mode]["jac_ms"].append(g.time_evaluations(a.evals, F, True))
            g.lm_iterations(1, F)
            t0 = time.perf_counter()
            s = g.lm_iterations(a.iters, F)
            res[mode]["lm_ms"].append((time.perf_counter() - t0) * 1e3 / max(1, s.iterations))
            g.close()
    for mode, v in res.items():
        j, m = np.array(v["jac_ms"]), np.array(v["lm_ms"])
        print(f"{mode:8s} Jacobian evaluation {np.median(j):.3f} ms (range {j.min():.3f}-{j.max():.3f}),"
              f" LM iteration {np.median(m):.3f} ms (range {m.min():.3f}-{m.max():.3f}) over {a.rounds} runs")


if __name__ == "__main__":
    main()
