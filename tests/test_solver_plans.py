"""Elimination plans of the damped normal-equation solve, on host-only handles (no GPU).

* The cases tests/test_gpu_solver.py checks against a dense reference cover every branch of the planner that selects different
  kernel code (P = 1 / odd / >= 64, uneven leaves, the smallest leaf, several reduction levels with odd block counts, border-only
  and border-free systems, border blocks in HBM, unstaged level-0 back-substitution, a grown level-0 window, a plan that does not fit).
* Where plans stop fitting: from a half bandwidth of 112 the level-0 window (256 slots) exceeds shared memory for any chunking, and a
  band too wide for several chunks leaves one chunk, whose back-substitution needs shared memory for every knot column.  Those shapes
  are refused when the problem is configured, with a message that names them.
* The reference and its bars can tell a subtly wrong solve from a right one.
"""
import numpy as np
import pytest

import solver_support as ss
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import calibrator
from openimucameracalibrator_b200 import synthetic as syn

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def _host(name, known_gravity=True):
    return ss.load(capi.CApi(calibrator.load_library(), "icc_", -1), name, known_gravity)


def _plans():
    out, handles = {}, {}
    for c in ss.CASES:
        key = (c.data, c.known_gravity)
        if key not in handles:
            handles[key] = _host(c.data, c.known_gravity)
        out[c.id] = handles[key].solver_plan(c.flags, c.chunks)
    h4 = _host("cfg4")
    for ch in ss.FULLSIZE_CHUNKS:
        out[f"cfg4-chunks{ch}"] = h4.solver_plan(ss.F_STAGE1, ch)
    out["points402"] = _host("points402").solver_plan(ss.F_POINTS)
    return out


@pytest.fixture(scope="module")
def plans():
    return _plans()


def test_gpu_cases_cover_every_plan_branch(plans):
    valid = [p for p in plans.values() if p["valid"]]
    banded = [p for p in valid if p["nk"] > 0]
    checks = {
        "P = 1": any(p["P"] == 1 for p in banded),
        "P odd > 1": any(p["P"] > 1 and p["P"] % 2 for p in banded),
        "P >= 64": any(p["P"] >= 64 for p in banded),
        "rem != 0": any(p["rem"] for p in banded),
        "rem == 0, P > 1": any(p["rem"] == 0 and p["P"] > 1 for p in banded),
        "smallest leaf kd + 1": any(p["P"] > 1 and p["len"] == p["kd"] + 1 for p in banded),
        "L >= 3": any(p["L"] >= 3 for p in banded),
        "odd block count at a reduction level": any(any(s % 2 and s > 1 for s in p["S"][:-1]) for p in banded),
        "nb = 0": any(p["nb"] == 0 for p in banded),
        "nk = 0": any(p["nk"] == 0 for p in valid),
        "cl_global": any(p["cl_global"] for p in banded),
        "cs_global": any(p["cs_global"] for p in valid),
        "stage0 = 0": any(not p["stage0"] for p in banded),
        "unstaged level-0 back-substitution": any(p["backsub0_staged"] < p["P"] for p in banded),
        "staged level-0 back-substitution": any(p["backsub0_staged"] == p["P"] for p in banded),
        "leaf > 128 columns": any(p["max_leaf"] > 128 for p in banded),
        "grown level-0 window": any(p["WS_A"] > 1 << (p["kd"] + 17 - 1).bit_length() for p in banded),
        "half bandwidth other than 35": any(p["kd"] not in (0, 35) for p in banded),
        "invalid plan": any(not p["valid"] for p in plans.values()),
    }
    assert all(checks.values()), [k for k, v in checks.items() if not v]


def test_plans_of_named_cases(plans):
    """Each case is named for the branch it is there for; this pins them, so that a planner change cannot silently move a case."""
    p = plans
    assert [p[f"cfg2-chunks{c}"]["P"] for c in (1, 2, 3, 4, 5, 7, 8, 16, 31)] == [1, 2, 3, 4, 5, 7, 8, 16, 17]
    assert p["cfg2-chunks-max"]["P"] == 17 and p["cfg2-chunks-max"]["L"] == 4          # the most chunks whose leaves keep kd + 1 columns
    assert p["cfg2-chunksauto"]["P"] == 16
    assert p["smallest-leaf"]["len"] == p["smallest-leaf"]["kd"] + 1
    assert p["nb0-spline"]["nb"] == 0 and p["nb1-spline-line-delay"]["nb"] == 1
    assert p["wide200-hbm-borders"]["cl_global"] and p["wide200-hbm-borders"]["cs_global"] and p["wide200-hbm-borders"]["nb"] >= 140
    pts = p["points396-unstaged"]
    assert pts["valid"] and pts["nb"] == 396 and not pts["stage0"] and pts["backsub0_staged"] == 0
    assert not p["points402"]["valid"] and p["points402"]["nb"] == 402
    for k in ("nk0-T_i_c", "nk0-line-delay", "nk0-gravity-acc-bias"):
        assert p[k]["nk"] == 0 and p[k]["valid"]
    assert p["kd47-dt-04-07"]["kd"] == p["kd47-dt-09-05"]["kd"] == 47
    assert p["kd62-two-chunks"]["kd"] == 62 and p["kd62-two-chunks"]["P"] == 2
    k110 = p["kd110-one-chunk"]
    assert k110["kd"] == 110 and k110["P"] == 1 and k110["max_leaf"] > 128 and k110["backsub0_staged"] == 0
    assert [p[f"cfg4-chunks{c}"]["P"] for c in ss.FULLSIZE_CHUNKS] == [128, 64, 127]
    assert p["P64-dense"]["P"] == 64 and p["P64-dense"]["rem"] > 0 and p["P64-dense"]["L"] == 5


def test_forced_chunks_match_the_partition(plans):
    """chunk c owns len + (c < rem) interior columns, P - 1 separators of kd columns between them; S halves level by level."""
    for k, p in plans.items():
        if not p["valid"] or p["nk"] == 0:
            continue
        w = p["kd"] if p["P"] > 1 else 0
        assert p["P"] * p["len"] + p["rem"] + (p["P"] - 1) * w == p["nk"], k
        assert 0 <= p["rem"] < p["P"] and (p["P"] == 1 or p["len"] >= p["kd"] + 1), k
        S = p["S"]
        assert S[0] == p["P"] - 1 and all(S[i + 1] == S[i] // 2 for i in range(len(S) - 1)) and S[-1] <= 1, k
        assert max(p["smem_bytes"]) <= 230000, k


def test_where_plans_stop_fitting():
    """Map the half bandwidth against the knot-spacing ratio and the sequence length, and turn the map into assertions."""
    lib = calibrator.load_library()
    seen = {}
    for so3 in np.round(np.arange(0.05, 0.1301, 0.0025), 4):
        for nf in ((60, 400, 3000) if so3 in (0.0625, 0.075, 0.0875, 0.1) else (60, 400)):
            h = capi.CApi(lib, "icc_", -1)
            capi.load_dataset(h, syn.make_dataset(syn.tiny_config(n_frames=nf, dt_so3_s=float(so3), dt_r3_s=0.02)))
            try:
                p = h.solver_plan(ss.F_STAGE1)
                seen[(so3, nf)] = ("ok", p["kd"], p["nk"], p)
            except capi.IccError as e:
                msg = str(e)
                assert "ICC_ERR_UNSUPPORTED" in msg and "half bandwidth of" in msg and "no elimination plan" in msg, msg
                kd = int(msg.split("half bandwidth of ")[1].split()[0]); nk = int(msg.split("over ")[1].split()[0])
                seen[(so3, nf)] = ("refused", kd, nk, None)
    ok = [v for v in seen.values() if v[0] == "ok"]
    refused = [v for v in seen.values() if v[0] == "refused"]
    # from kd 112 nothing fits; every accepted shape has a valid plan for its actual border
    assert all(kd < 112 for _, kd, _, _ in ok) and any(kd >= 112 for _, kd, _, _ in refused)
    assert all(p["valid"] for *_, p in ok)
    # several chunks stop fitting far below that: the widest multi-chunk band is kd 62 (the reduced systems' fronts are 3 kd wide)
    multi = [kd for _, kd, _, p in ok if p["P"] > 1]
    assert max(multi) == 62 and all(p["P"] == 1 for _, kd, _, p in ok if kd > 62)
    # one chunk over a long sequence: the back-substitution keeps every knot column in shared memory, so every band too wide for
    # several chunks has a length limit, single_chunk_max_columns(kd) (15 076 columns at kd 68, 2 182 at kd 110); the message names it
    for status, kd, nk, p in seen.values():
        if 62 < kd < 112:
            assert (status == "ok") == (nk <= ss.single_chunk_max_columns(kd)), (status, kd, nk)
    assert any(62 < kd < 80 and nk > 15000 for s, kd, nk, _ in refused) and any(kd >= 107 and nk < 500 for _, kd, nk, _ in ok)


@pytest.mark.parametrize("data,flags,where", ss.UNFIT, ids=[u[0] for u in ss.UNFIT])
def test_unfit_shapes_are_refused_with_an_accurate_message(data, flags, where):
    h = _host(data)
    if where == "configure":
        with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED.*half bandwidth of [0-9]+ columns.*no elimination plan") as e:
            h.num_tangent(flags)
        kd = int(str(e.value).split("half bandwidth of ")[1].split()[0])
        if kd < 112:
            assert f"takes at most {ss.single_chunk_max_columns(kd)} knot columns" in str(e.value)
        else:
            assert "at any sequence length" in str(e.value)
    else:
        p = h.solver_plan(flags)                                        # the border alone does not fit: evaluation still works
        assert not p["valid"] and p["nb"] > 400


# ---- the reference can tell a subtly wrong solve from a right one ------------------------------------------------------------
def test_refused_shape_leaves_the_configured_layout_intact():
    """A refused configuration must not leave its layout behind: the previously configured flags keep their tangent count and plan."""
    h = _host("kd113")
    n_ld, plan_ld = h.num_tangent(ss.F_STAGE2), h.solver_plan(ss.F_STAGE2)
    assert n_ld == 1 and plan_ld["nk"] == 0 and plan_ld["nb"] == 1
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED"):
        h.num_tangent(ss.F_STAGE1)
    assert h.num_tangent(ss.F_STAGE2) == n_ld and h.solver_plan(ss.F_STAGE2) == plan_ld
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED"):
        h.solver_plan(ss.F_STAGE1)
    assert h.solver_plan(ss.F_STAGE2) == plan_ld and h.num_tangent(ss.F_STAGE2) == n_ld


@pytest.mark.parametrize("data,flags,known_gravity", [("tiny", ss.F_STAGE1, True), ("tiny", ss.F_ALL, False), ("dt_04_07", ss.F_STAGE1, True)],
                         ids=["tiny-stage1", "tiny-all-biases", "kd47"])
def test_reference_bars_catch_a_1e9_coupling_error(oracle_factory, data, flags, known_gravity):
    """On the real normal equations (the CPU oracle's H and g of the same dataset) at the LM's initial radius: the reference meets both
    bars by two decades, and a solve that got one coupling entry wrong by 1e-9 relative exceeds both bars at least 100-fold -- for a
    separator - interior entry, a border entry and an entry across a chunk boundary of the plan the solver uses."""
    o = ss.load(oracle_factory(), data, known_gravity)
    _, _, g, H = o.evaluate(flags, residuals=False, hessian=True)
    plan = _host(data, known_gravity).solver_plan(flags)
    nk, kd, nb = plan["nk"], plan["kd"], plan["nb"]
    assert plan["P"] >= 2 or nb > 0
    sys_ = ss.lm_system(H, g, 1e4)
    ref = ss.reference(sys_)
    assert ss.backward_error(sys_, ref.y) <= ref.eta_bar / 100 and ss.componentwise_error(sys_, ref.y) <= ref.omega_bar / 100
    # plain float64 Cholesky without refinement is inside the bars too: they are what a backward-stable solve meets
    y0 = ss.cholesky_solve(sys_)
    assert ss.backward_error(sys_, y0) <= ref.eta_bar and ss.componentwise_error(sys_, y0) <= ref.omega_bar
    cases = {"border": ss.strongest_coupling(sys_, ref.y, np.arange(nk, nk + nb), np.arange(nk))}
    if plan["P"] >= 2:
        a1 = plan["len"] + (1 if plan["rem"] else 0)          # chunk 0 interior [0, a1), separator [a1, a1 + kd), chunk 1 from a1 + kd
        sep, left, right = np.arange(a1, a1 + kd), np.arange(max(0, a1 - kd), a1), np.arange(a1 + kd, min(nk, a1 + 2 * kd))
        cases["separator-interior"] = ss.strongest_coupling(sys_, ref.y, sep, left)
        cases["across-chunk-boundary"] = ss.strongest_coupling(sys_, ref.y, right, sep)
    for name, (i, j) in cases.items():
        yw = ss.perturbed_solution(sys_, i, j, 1e-9)
        eta_w, omega_w = ss.backward_error(sys_, yw), ss.componentwise_error(sys_, yw)
        assert eta_w >= 100 * ref.eta_bar, (name, i, j, eta_w, ref.eta_bar)
        assert omega_w >= 100 * ref.omega_bar, (name, i, j, omega_w, ref.omega_bar)


def test_reference_model_change_and_scale():
    H, g = ss.banded_bordered_hessian(120, 35, 6, seed=9)
    sys_ = ss.lm_system(H, g, 1e2)
    ref = ss.reference(sys_)
    assert np.array_equal(sys_.s, 1.0 / (1.0 + np.sqrt(np.diag(H))))
    y = ref.y
    m_solver = 0.5 * float(np.sum(sys_.dlm * y * y) + np.dot(y, sys_.b))      # the solver's form (y^T D y - y^T S g) / 2
    assert abs(m_solver - ss.model_change(H, g, ref.delta)) <= ss.model_change_bar(sys_, y, ref.eta_bar)


def test_plus_statement_small_cases():
    """The NumPy Plus: SE(3) exp at zero rotation equals a pure translation; SO(3) right-exp composes; the bias box clips."""
    q, t = ss.se3_exp([0.1, -0.2, 0.3, 0, 0, 0])
    assert np.allclose(q, [0, 0, 0, 1]) and np.allclose(t, [0.1, -0.2, 0.3])
    q1 = ss.so3_exp_quat([0.3, 0, 0])
    assert np.allclose(ss._qmul(q1, q1), ss.so3_exp_quat([0.6, 0, 0]))
    layout = dict(spline=False, tic=False, gravity=False, line_delay=False, acc_bias=False, gyr_bias=True)
    st = (np.zeros((0, 4)), np.zeros((0, 3)), np.zeros((0, 3)), np.array([[0.09, 0.0, -0.05]]), np.zeros(7), np.zeros(3), 0.0)
    out = ss.plus(st, np.array([0.05, 0.01, -0.1]), layout)
    assert np.allclose(out[3], [[0.1, 0.01, -0.1]])
