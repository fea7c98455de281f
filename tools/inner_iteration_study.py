#!/usr/bin/env python
"""Where does ceres' use_inner_iterations (spline_trajectory_estimator.impl.h:266) move the reference's stopping point?

Runs the CPU oracle three ways on BASELINE configs (both stages of the hot CLI: SPLINE | T_I_C, then CAM_LINE_DELAY):
  plain   : the LM path the CUDA product follows (function_tolerance 1e-4, parameter_tolerance 1e-7 -- impl.h:263-264),
  inner   : the same with Ceres' inner iterations restated (oracle/icc_oracle.cpp: inner_iterations),
  optimum : plain LM with tolerances 1e-12 (the true minimiser both paths head for).
Prints one JSON line per config.
usage: python tools/inner_iteration_study.py 1 2 3"""
import ctypes as C, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from openimucameracalibrator_b200 import _capi as capi, synthetic as syn
from oracle_api import new_oracle, oracle_lib

F1 = capi.FLAG_SPLINE | capi.FLAG_T_I_C; F2 = capi.FLAG_CAM_LINE_DELAY
lib = oracle_lib()
lib.icco_set_inner_iterations.argtypes = [C.c_void_p, C.c_int]; lib.icco_inner_iteration_steps.argtypes = [C.c_void_p]


def run(ds, inner, tight=False):
    o = new_oracle(); capi.load_dataset(o, ds)
    lib.icco_set_inner_iterations(o.h, int(inner))
    if tight:
        o.set_solver_options(function_tolerance=1e-12, parameter_tolerance=1e-12)
    t0 = time.time(); s1 = o.optimize(100 if tight else 50, F1); n_in = lib.icco_inner_iteration_steps(o.h); s2 = o.optimize(50 if tight else 10, F2)
    return dict(lm_iterations=s1.iterations, termination=s1.termination, cost_stage1=s1.final_cost, inner_iteration_steps=n_in, lm_iterations_stage2=s2.iterations,
                T_i_c=o.get_T_i_c().tolist(), line_delay=o.get_line_delay(), reproj_px=s2.mean_reproj_error, seconds=time.time() - t0)


def rel(x, y):
    return float(np.abs(np.array(x) - np.array(y)).max() / np.abs(np.array(y)).max())


if __name__ == "__main__":
    for c in [int(a) for a in sys.argv[1:]] or [1, 2]:
        ds = syn.make_dataset(syn.CONFIGS[c])
        a, b, t = run(ds, False), run(ds, True), run(ds, False, tight=True)
        print(json.dumps(dict(config=c, plain=a, inner=b, optimum=t,
                              rel_T_i_c=dict(inner_vs_plain=rel(b["T_i_c"], a["T_i_c"]), plain_vs_optimum=rel(a["T_i_c"], t["T_i_c"]), inner_vs_optimum=rel(b["T_i_c"], t["T_i_c"])),
                              rel_line_delay=dict(inner_vs_plain=abs(b["line_delay"] - a["line_delay"]) / abs(a["line_delay"]), plain_vs_optimum=abs(a["line_delay"] - t["line_delay"]) / abs(t["line_delay"]),
                                                  inner_vs_optimum=abs(b["line_delay"] - t["line_delay"]) / abs(t["line_delay"])),
                              truth=dict(T_i_c=ds["truth"]["T_i_c"].tolist(), line_delay=ds["truth"]["line_delay"]))), flush=True)
