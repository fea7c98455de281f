"""Developer probe (not a test): legacy vs persistent vision kernel on the BASELINE configs -- parity of cost / gradient / LM step and timings."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn
F = capi.FLAG_SPLINE | capi.FLAG_T_I_C
cfgs = [int(a) for a in sys.argv[1:]] or [4, 3, 2, 1]
for c in cfgs:
    ds = syn.make_dataset(syn.CONFIGS[c])
    out = {}
    for variant in ("legacy", "tmem"):
        if variant == "legacy": os.environ["ICC_VISION_LEGACY"] = "1"; os.environ["ICC_IMU_LEGACY"] = "1"
        else: os.environ.pop("ICC_VISION_LEGACY", None); os.environ.pop("ICC_IMU_LEGACY", None)
        g = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(g, ds)
        cost, r, grad, _ = g.evaluate(F, residuals=True, gradient=True, hessian=False)
        g.time_evaluations(3, F, 2)
        vis = g.time_evaluations(20, F, 2); jac = g.time_evaluations(20, F, 1); imu = g.time_evaluations(20, F, 3)
        s = g.lm_iterations(3, F)
        out[variant] = (cost, r, grad, s.final_cost, g.get_T_i_c())
        print(f"cfg{c} {variant:6s}: vision {vis*1e3:7.1f} us  imu {imu*1e3:6.1f} us  jac {jac*1e3:7.1f} us | lm3: jac_in_lm {1e6*s.seconds_jacobian/max(1,s.jacobian_evaluations):6.1f} us solve {1e6*s.seconds_linear_solve/s.iterations:6.1f} us/iter wall {s.seconds_total*1e3:.2f} ms cost {s.final_cost:.9e}", flush=True)
    a, b = out["legacy"], out["tmem"]
    rel = lambda x, y: float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-300))
    print(f"cfg{c} parity tmem vs legacy: cost {abs(a[0]-b[0])/abs(a[0]):.2e} residuals {rel(a[1], b[1]):.2e} gradient {rel(a[2], b[2]):.2e} lm3 cost {abs(a[3]-b[3])/abs(a[3]):.2e} T_i_c {rel(a[4], b[4]):.2e}", flush=True)
