"""Developer probe (not a test): lockstep groups / stagger of the persistent evaluation kernel on config 4.  python tests/stagger_probe.py"""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn
F = capi.FLAG_SPLINE | capi.FLAG_T_I_C
ds = syn.make_dataset(syn.CONFIGS[int(sys.argv[1]) if len(sys.argv) > 1 else 4])
g = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(g, ds)
ref = None
for name, env in [("groups 1", {"ICC_TMEM_GROUPS": "1"}), ("groups 2", {"ICC_TMEM_GROUPS": "2"}), ("groups 3", {"ICC_TMEM_GROUPS": "3"}), ("groups 4", {"ICC_TMEM_GROUPS": "4"}),
                  ("groups 6", {"ICC_TMEM_GROUPS": "6"}), ("no lockstep", {"ICC_TMEM_NO_LOCKSTEP": "1"}), ("default", {}), ("groups 1", {"ICC_TMEM_GROUPS": "1"})]:
    for k in ("ICC_TMEM_GROUPS", "ICC_TMEM_STAGGER_NS", "ICC_TMEM_NO_LOCKSTEP"): os.environ.pop(k, None)
    os.environ.update(env)
    cost, _, grad, _ = g.evaluate(F, residuals=False)
    if ref is None: ref = (cost, grad)
    g.time_evaluations(3, F, 1)
    vis = min(g.time_evaluations(20, F, 2) for _ in range(3)); imu = min(g.time_evaluations(20, F, 3) for _ in range(3)); jac = min(g.time_evaluations(20, F, 1) for _ in range(3))
    print(f"{name:14s}: vision {vis*1e3:7.1f} us  imu {imu*1e3:6.1f} us  jac {jac*1e3:7.1f} us   parity cost {abs(cost-ref[0])/ref[0]:.1e} grad {np.abs(grad-ref[1]).max()/np.abs(ref[1]).max():.1e}", flush=True)
