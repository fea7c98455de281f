"""Developer probe (not a test): schedule variants of the unified persistent evaluation kernel on BASELINE config 4 / 3."""
import sys, os, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
code = r'''
import sys, os
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, "tests"))
from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn
F = capi.FLAG_SPLINE | capi.FLAG_T_I_C
for c in (4, 3):
    ds = syn.make_dataset(syn.CONFIGS[c])
    g = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(g, ds)
    g.time_evaluations(3, F, 1)
    print("cfg", c, os.environ.get("ICC_IMU_COST"), "vision_first" if os.environ.get("ICC_TMEM_VISION_FIRST") else "imu_first", "jac %%.1f us" %% (1e3 * g.time_evaluations(20, F, 1)), flush=True)
''' % (ROOT, ROOT)
for cost in ("1.6", "2.4", "3.2"):
    for vf in (None, "1"):
        env = dict(os.environ); env["ICC_IMU_COST"] = cost
        if vf: env["ICC_TMEM_VISION_FIRST"] = "1"
        subprocess.run([sys.executable, "-c", code], env=env)
