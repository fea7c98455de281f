"""Cost of FISHEYE_RADIAL_TANGENTIAL's persistent-kernel instantiation: BASELINE config 4's sequence (3000 views x 144 corners) projected
through a decentred Kannala-Brandt lens with six radial and two tangential terms, against the same sequence in FISHEYE (k1..k4).  For each model, in alternating rounds on fresh handles:
  * the whole Jacobian evaluation (icc_time_evaluations: CUDA events around n evaluations);
  * the persistent vision launch alone, eval_tmem_kernel<model> (torch.profiler with CUDA activities around the same evaluations, in a
    separate pass so that tracing does not slow the timed one).
Prints the card, its power limit and its SM clock with the numbers.
usage: python tools/fisheye_radtan_timing.py [--rounds 4] [--evals 20]"""
import argparse
import dataclasses
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from openimucameracalibrator_b200 import _capi as capi, calibrator, camera_models as cm, synthetic as syn  # noqa: E402

F = capi.FLAG_SPLINE | capi.FLAG_T_I_C
# the config's focal length and principal point; a wide lens with all six radial terms and off-centre tangential terms (its domain test
# isolates the roots of d theta_d / d theta per corner), and the same k1..k4 for FISHEYE
FISHEYE_RADTAN_K = (438.0, 1.0, 0.0, 489.5, 272.0, 0.02, -0.004, 6e-4, -5e-5, 2e-6, -3e-8, 1.2e-3, -8e-4)
FISHEYE_K = FISHEYE_RADTAN_K[:9]


def vision_kernel_us(g, n):
    """mean device time of eval_tmem_kernel<model> per evaluation over n evaluations, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.time_evaluations(n, F, True)
    tot, cnt = 0.0, 0
    for e in prof.key_averages():
        if "eval_tmem_kernel" in e.key and "ILin" not in e.key and "<-" not in e.key:     # the vision instantiations, not the IMU ones (<-1>, <-2>)
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)); cnt += e.count
    return tot / n if cnt else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--evals", type=int, default=20)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    cfg4 = syn.CONFIGS[4]
    data = {"FISHEYE": syn.make_dataset(dataclasses.replace(cfg4, name="cfg4_fisheye_3000x144", model=cm.FISHEYE, intrinsics=FISHEYE_K)),
            "FISHEYE_RADIAL_TANGENTIAL": syn.make_dataset(dataclasses.replace(cfg4, name="cfg4_fisheye_radtan_3000x144", model=cm.FISHEYE_RADIAL_TANGENTIAL,
                                                                              intrinsics=FISHEYE_RADTAN_K))}
    lib = calibrator.load_library()
    res = {m: {"jac_ms": [], "vision_us": []} for m in data}
    for r in range(a.rounds):
        for m in (list(data) if r % 2 == 0 else list(data)[::-1]):
            g = capi.CApi(lib, "icc_", 0)
            capi.load_dataset(g, data[m])
            g.time_evaluations(3, F, True)                                  # warm-up: modules, allocations, layout
            res[m]["jac_ms"].append(g.time_evaluations(a.evals, F, True))
            res[m]["vision_us"].append(vision_kernel_us(g, a.evals))
            g.close()
    for m, v in res.items():
        j, k = np.array(v["jac_ms"]), np.array(v["vision_us"])
        print(f"{m:25s} Jacobian evaluation {np.median(j):.3f} ms (range {j.min():.3f}-{j.max():.3f}), persistent vision launch"
              f" {np.median(k):.1f} us (range {k.min():.1f}-{k.max():.1f}) over {a.rounds} runs")


if __name__ == "__main__":
    main()
