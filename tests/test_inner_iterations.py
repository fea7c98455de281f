"""Ceres' use_inner_iterations = true (spline_trajectory_estimator.impl.h:266), restated in the oracle (oracle/icc_oracle.cpp:
inner_iterations -- CoordinateDescentMinimizer over recursive independent sets + TrustRegionMinimizer::DoInnerIterationsIfNeeded).

The CUDA product runs plain Levenberg-Marquardt.  What these tests pin: the refinement really is a descent step of the same
objective, it heads for the SAME minimiser (so parity "at the true optimum" -- SURVEY §7 -- is the meaningful comparison), and at
the reference's loose function_tolerance = 1e-4 BOTH stopping points sit further from that minimiser than they sit from each other
times a small factor: the reference's own stopping point is not defined to 1e-4 (tools/inner_iteration_study.py prints the
numbers for BASELINE configs 1-3)."""
import ctypes as C

import numpy as np

from helpers import F_STAGE1, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn
from oracle_api import new_oracle, oracle_lib


def _oracle(ds, inner, **opts):
    lib = oracle_lib()
    lib.icco_set_inner_iterations.argtypes = [C.c_void_p, C.c_int]; lib.icco_inner_iteration_steps.argtypes = [C.c_void_p]
    o = new_oracle(); capi.load_dataset(o, ds)
    lib.icco_set_inner_iterations(o.h, int(inner))
    if opts:
        o.set_solver_options(**opts)
    return o, lib


def test_inner_iterations_are_a_descent_refinement_of_the_same_objective():
    ds = syn.make_dataset(syn.tiny_config(n_frames=30))
    a, _ = _oracle(ds, False); b, lib = _oracle(ds, True)
    sa, sb = a.lm_iterations(1, F_STAGE1), b.lm_iterations(1, F_STAGE1)
    assert lib.icco_inner_iteration_steps(b.h) == 1
    assert sb.initial_cost == sa.initial_cost and sb.final_cost < sa.final_cost          # same start, lower cost after the refinement
    assert abs(b.evaluate(F_STAGE1, gradient=False)[0] - sb.final_cost) <= 1e-12 * sb.final_cost   # the reported cost is the cost of the state


def test_inner_iterations_switch_themselves_off():
    """inner_iteration_tolerance = 1e-3: once a refinement gains less than that relative to the candidate cost, Ceres stops refining."""
    ds = syn.make_dataset(syn.tiny_config(n_frames=30))
    b, lib = _oracle(ds, True, function_tolerance=1e-13, parameter_tolerance=1e-13)
    sb = b.optimize(60, F_STAGE1)
    assert 0 < lib.icco_inner_iteration_steps(b.h) < sb.iterations


def test_reference_tolerance_leaves_the_stopping_point_undetermined_at_1e_4():
    """BASELINE config 1 with the reference's own tolerances: the stopping points with and without inner iterations differ by a few
    1e-3 relative in T_i_c (1-2 mm of the weakly observable lever arm) -- an order of magnitude above the north-star's 1e-4, while
    the GPU path reproduces the plain path to 1e-8 (tests/test_gpu_lm.py).  The numbers for configs 1-3, next to the tight-tolerance
    runs, come from tools/inner_iteration_study.py."""
    ds = syn.make_dataset(syn.CONFIGS[1])
    a, _ = _oracle(ds, False); b, lib = _oracle(ds, True)
    sa, sb = a.optimize(50, F_STAGE1), b.optimize(50, F_STAGE1)
    assert sa.termination == 1 and sb.termination == 1 and lib.icco_inner_iteration_steps(b.h) >= 1
    assert sb.final_cost < sa.final_cost
    d_ab = rel(a.get_T_i_c(), b.get_T_i_c())
    assert 1e-4 < d_ab < 2e-2, d_ab
    qa, qb = a.get_T_i_c()[:4], b.get_T_i_c()[:4]
    assert np.degrees(2 * np.arccos(min(1.0, abs(float(qa @ qb))))) < 0.1          # the rotation barely moves; the lever arm does
