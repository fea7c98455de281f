"""The nested-dissection LM solve (icc_solve_normal_equations) against a dense float64 Cholesky with long-double iterative refinement
of exactly the H and g that were factored (tests/solver_support.py), over every branch of the elimination planner.

Per case: the plan the solve used equals icc_solver_plan's; the Jacobi scale equals 1/(1+sqrt(H_ii)) of the returned diagonal bit
for bit; the normwise and componentwise backward errors are within their bars; the forward error is within 4 kappa eta_bar; the model
cost change matches -(g^T delta + delta^T H delta / 2).  Config 4 runs at full size through J^T J products, and one LM iteration must
land exactly on Plus(x, delta) of the solved step."""
import numpy as np
import pytest

import solver_support as ss
from openimucameracalibrator_b200 import _capi as capi

pytestmark = pytest.mark.gpu


def _handle(gpu_factory, data, known_gravity=True, jacobi=1):
    g = ss.load(gpu_factory(), data, known_gravity)
    if not jacobi:
        g.set_solver_options(jacobi_scaling=0)
    return g


def _check_dense(g, case):
    cost, _, grad, H = g.evaluate(case.flags, residuals=False, hessian=True)
    predicted = g.solver_plan(case.flags, case.chunks)
    launches = capi.kernel_launch_count(g.lib)
    out = g.solve_normal_equations(case.flags, case.radius, case.chunks)
    assert capi.kernel_launch_count(g.lib) > launches
    assert out["plan"] == predicted
    assert out["step_ok"] == 1
    assert np.array_equal(out["h_diag"], np.diag(H))
    s_ref = 1.0 / (1.0 + np.sqrt(out["h_diag"])) if case.jacobi else np.ones_like(out["h_diag"])
    assert np.array_equal(out["scale"], s_ref)
    sys_ = ss.lm_system(H, grad, case.radius, case.jacobi)
    ref = ss.reference(sys_)
    y = out["delta"] / sys_.s
    eta, omega = ss.backward_error(sys_, y), ss.componentwise_error(sys_, y)
    fwd = float(np.abs(y - ref.y).max() / np.abs(ref.y).max())
    dm = abs(out["model_change"] - ss.model_change(H, grad, out["delta"]))
    dm_bar = ss.model_change_bar(sys_, y, ref.eta_bar)
    print(f"SOLVER-METRICS {case.id}: n={len(y)} P={out['plan']['P']} kd={out['plan']['kd']} nb={out['plan']['nb']} eta={eta:.2e} "
          f"(bar {ref.eta_bar:.2e}) omega={omega:.2e} (bar {ref.omega_bar:.2e}) fwd={fwd:.2e} kappa={ref.kappa:.2e} dm={dm:.2e} (bar {dm_bar:.2e})")
    assert eta <= ref.eta_bar, (eta, ref.eta_bar)
    assert omega <= ref.omega_bar, (omega, ref.omega_bar)
    if ref.kappa * ss.EPS <= 1e-2:
        assert fwd <= 4 * ref.kappa * ref.eta_bar, (fwd, ref.kappa)
    assert dm <= dm_bar, (out["model_change"], dm, dm_bar)
    return out, ref


@pytest.mark.parametrize("case", ss.CASES, ids=[c.id for c in ss.CASES])
def test_solve_matches_dense_reference(gpu_factory, case):
    g = _handle(gpu_factory, case.data, case.known_gravity, case.jacobi)
    _check_dense(g, case)


def test_unfit_border_is_refused_before_any_launch(gpu_factory):
    """402 border columns (132 board points next to T_i_c): no plan; evaluation works, the solve refuses with nothing launched and
    the handle stays usable."""
    g = _handle(gpu_factory, "points402")
    g.evaluate(ss.F_POINTS, residuals=False)
    launches = capi.kernel_launch_count(g.lib)
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED.*border of 402 columns"):
        g.solve_normal_equations(ss.F_POINTS, 1e4)
    assert capi.kernel_launch_count(g.lib) == launches
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED.*border of 402 columns"):
        g.lm_iterations(1, ss.F_POINTS)
    assert g.lm_iterations(1, ss.F_STAGE1).successful_steps == 1


def test_solve_needs_current_normal_equations(gpu_factory):
    g = _handle(gpu_factory, "tiny")
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        g.solve_normal_equations(ss.F_STAGE1, 1e4)
    g.evaluate(ss.F_STAGE1, residuals=False)
    g.solve_normal_equations(ss.F_STAGE1, 1e4)
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        g.solve_normal_equations(ss.F_ALL, 1e4)          # other flags
    g.lm_iterations(1, ss.F_STAGE1)                      # moves the state and re-evaluates
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        g.solve_normal_equations(ss.F_STAGE1, 1e4)


@pytest.fixture(scope="module")
def cfg4(cuda_lib):
    g = ss.load(capi.CApi(cuda_lib, "icc_", 0), "cfg4")
    yield g
    g.close()


@pytest.mark.parametrize("chunks", ss.FULLSIZE_CHUNKS)
def test_fullsize_config4(cfg4, chunks):
    """Config 4 at full size: eta and the model change through J^T J products of a fresh evaluation.  The products carry that
    evaluation's own rounding (atomics), of the order of u ||A|| ||y||, inside the bar.  Without a factor the growth rho of the bar is
    unknown; the check takes rho = 1, the smallest value it can have (|L||L^T| >= |A| entrywise), so the bar used is never looser than
    the analysed one.  The sensitive check of the 64-chunk branch is the dense case P64-dense."""
    g, f = cfg4, ss.F_STAGE1
    _, _, grad, _ = g.evaluate(f, residuals=False)
    out = g.solve_normal_equations(f, 1e4, chunks)
    assert out["plan"] == g.solver_plan(f, chunks) and out["step_ok"] == 1
    assert out["plan"]["P"] == {0: 128, 64: 64, 127: 127}[chunks]
    s, hd, delta = out["scale"], out["h_diag"], out["delta"]
    assert np.array_equal(s, 1.0 / (1.0 + np.sqrt(hd)))
    dlm = np.clip(hd * s * s, 1e-6, 1e32) / 1e4
    y = delta / s
    ones = np.ones_like(delta)
    Hd, H1, Hs = g.normal_matvec(f, np.stack([delta, s, s * np.sign(y)]))
    r = s.astype(np.longdouble) * Hd + dlm * y.astype(np.longdouble) + s.astype(np.longdouble) * grad
    # ||A||_inf from below (|A v|_inf for |v| = 1): the estimate only makes eta larger
    nA = max(float(np.abs(s * H1 + dlm * ones).max()), float(np.abs(s * Hs + dlm * np.sign(y)).max()), float(np.max(hd * s * s + dlm)))
    b = -s * grad
    eta = float(np.abs(r).max()) / (nA * float(np.abs(y).max()) + float(np.abs(b).max()))
    bar = ss.eta_bar(len(y), 1.0)
    m_ref = float(-(np.asarray(grad, np.longdouble) @ np.asarray(delta, np.longdouble) + 0.5 * (np.asarray(delta, np.longdouble) @ Hd)))
    terms = float(np.sum(dlm * y * y + np.abs(y * b)))
    dm_bar = 0.5 * float(np.abs(y).sum()) * bar * (nA * float(np.abs(y).max()) + float(np.abs(b).max())) + 2 * (len(y) + 4) * ss.U * terms
    print(f"SOLVER-METRICS cfg4-chunks{chunks}: n={len(y)} P={out['plan']['P']} L={out['plan']['L']} eta={eta:.2e} (bar {bar:.2e}) "
          f"dm={abs(out['model_change'] - m_ref):.2e} (bar {dm_bar:.2e})")
    assert eta <= bar
    assert abs(out["model_change"] - m_ref) <= dm_bar


def test_step_into_state(gpu_factory):
    """lm_iterations(1) from a state equals Plus(state, delta) of the step solved at the initial radius: SO(3) right-exp, R^3
    addition, SE(3) exp on T_i_c, gravity, line delay and the bias box -- with one gyroscope bias knot pushed across its box."""
    f = ss.F_ALL
    g = _handle(gpu_factory, "tiny", known_gravity=False)
    g.evaluate(f, residuals=False)
    d0 = g.solve_normal_equations(f, 1e4)["delta"]
    nso3, nr3, nba, nbg = g.num_knots()
    c_bg = 3 * nso3 + 3 * nr3 + 6 + 3 + 1 + 3 * nba
    so3, r3, ba, bg = g.get_knots()
    k = int(np.argmax(np.abs(d0[c_bg:c_bg + 3 * nbg])))
    bg = bg.copy()
    bg.flat[k] = np.sign(d0[c_bg + k]) * (0.1 - 0.25 * abs(d0[c_bg + k]))     # the step crosses the box by about 3/4 of itself
    g.set_knots(bg=bg)
    state = (*g.get_knots(), g.get_T_i_c(), g.get_gravity(), g.get_line_delay())
    g.evaluate(f, residuals=False)
    delta = g.solve_normal_equations(f, 1e4)["delta"]
    assert abs(state[3].flat[k] + delta[c_bg + k]) > 0.1
    s = g.lm_iterations(1, f)
    assert s.successful_steps == 1
    layout = dict(spline=True, tic=True, gravity=True, line_delay=True, acc_bias=True, gyr_bias=True)
    want = ss.plus(state, delta, layout)
    got = (*g.get_knots(), g.get_T_i_c(), g.get_gravity(), g.get_line_delay())
    # lm_iterations evaluates H and g once more (atomics: other last bits), so its step differs from delta by ~kappa u |delta|
    tol = 1e-7 * float(np.abs(delta).max()) + 1e-14
    for name, a, b in zip(("so3", "r3", "ba", "bg", "T_i_c", "gravity", "line_delay"), got, want):
        assert np.abs(np.asarray(a) - np.asarray(b)).max() <= tol, name
    assert abs(got[3].flat[k]) == 0.1
