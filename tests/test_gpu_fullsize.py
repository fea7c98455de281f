"""BASELINE.json full-size configurations against the oracle AT FULL SIZE (the oracle's evaluation runs on every host core through a
persistent pool; config 4 = 1.46 M residuals takes well under a second per Jacobian evaluation on the GPU box):
  * config 4: cost, J^T r and J^T J (through products with random vectors: every stored entry of the banded + bordered system) at 1e-9,
    the state after one LM iteration, and the whole LM run (same iteration count, T_i_c to 1e-8);
  * config 3 (DoubleSphere, 1000 x 96, 400 Hz): both stages on ALL frames, line delay to 1e-7.
Plus size-independent properties of config 4:
  (1) cost from the Jacobian kernels == cost from the cost-only kernels,
  (2) J^T r agrees with directional finite differences of the GPU cost,
  (3) residual shards are additive: sum over time-slice shards of (cost, J^T r) == unsharded,
  (4) an oracle spot check on a strided subset of residuals (value parity of the same kernels at full size),
  (5) LM reduces the cost and the model/actual decrease ratio of an accepted step is sane."""
import numpy as np
import pytest

from helpers import F_STAGE1, TangentWalker, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_block_probes, probe_reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ds4():
    return syn.make_dataset(syn.CONFIGS[4])


def test_config4_shape(gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    assert g.num_knots()[:2] == (2005, 2005)
    nv, na, ng = g.num_residuals()
    assert nv == 864000 and abs(na - 299901) < 10 and na == ng
    assert g.num_tangent(F_STAGE1) == 12036


def test_config4_cost_paths_and_gradient_fd(gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    c_jac, _, grad, _ = g.evaluate(F_STAGE1, residuals=False)
    c_only = g.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    assert abs(c_jac - c_only) <= 1e-11 * c_only
    w = TangentWalker(g, F_STAGE1)
    rng = np.random.default_rng(4)
    d = rng.normal(size=w.n); eps = 1e-7
    fd = (w.cost(eps * d) - w.cost(-eps * d)) / (2 * eps)
    assert abs(fd - grad @ d) <= 1e-5 * abs(fd)


def test_config4_shards_are_additive(gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    c, _, grad, _ = g.evaluate(F_STAGE1, residuals=False)
    cs, gs, nres = 0.0, 0.0, 0
    for r in range(4):
        s = gpu_factory(); capi.load_dataset(s, ds4, shard=(r, 4))
        ci, _, gi, _ = s.evaluate(F_STAGE1, residuals=False)
        cs += ci; gs = gs + gi; nres += sum(s.num_residuals())
        s.close()
    assert nres == sum(g.num_residuals())
    assert abs(cs - c) <= 1e-11 * c and rel(gs, grad) < 1e-10


def test_config4_residual_spot_check_against_oracle(oracle_factory, gpu_factory, ds4):
    """The oracle evaluates residual VALUES of the full problem in well under a second (no Jacobians)."""
    g = gpu_factory(); capi.load_dataset(g, ds4)
    o = oracle_factory(); capi.load_dataset(o, ds4)
    cg, rg, _, _ = g.evaluate(F_STAGE1, gradient=False)
    co, ro, _, _ = o.evaluate(F_STAGE1, gradient=False)
    assert rel(rg, ro) < 1e-9 and abs(cg - co) <= 1e-10 * co


def test_config4_lm_step(gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    s = g.lm_iterations(2, F_STAGE1)
    assert s.successful_steps >= 1 and s.final_cost < 0.05 * s.initial_cost
    s = g.optimize(50, F_STAGE1)
    assert s.termination in (1, 2) and 0.15 < s.mean_reproj_error < 0.4
    q = g.get_T_i_c(); qt = ds4["truth"]["T_i_c"]
    assert np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4]))))) < 0.05
    assert np.linalg.norm(q[4:] - qt[4:]) < 1e-2      # function_tolerance 1e-4 stops early (same as the reference); init was 2.3 cm off


# ---- full-size oracle parity (VERDICT r1 item 2: the north-star's acceptance sentence at the size it is quoted on) -------------------------
def test_config4_jacobian_parity_against_oracle(oracle_factory, gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    o = oracle_factory(); capi.load_dataset(o, ds4)
    cg, _, gg, _ = g.evaluate(F_STAGE1, residuals=False)
    co, _, go, _ = o.evaluate(F_STAGE1, residuals=False)
    assert abs(cg - co) <= 1e-10 * co
    assert rel(gg, go) < 1e-9
    rng = np.random.default_rng(44)
    n = g.num_tangent(F_STAGE1)
    V = rng.normal(size=(4, n)); V[1, : n - 6] = 0.0; V[2, n - 6:] = 0.0      # all columns / border only / band only / all
    Hg, Ho = g.normal_matvec(F_STAGE1, V), o.normal_matvec(F_STAGE1, V)
    for a, b in zip(Hg, Ho):
        assert rel(a, b) < 1e-9
    assert_block_probes(g, probe_reference(o, F_STAGE1, rng))       # each column block and the end knots at their own scale


def test_config4_lm_parity_against_oracle(oracle_factory, gpu_factory, ds4):
    g = gpu_factory(); capi.load_dataset(g, ds4)
    o = oracle_factory(); capi.load_dataset(o, ds4)
    s1g, s1o = g.lm_iterations(1, F_STAGE1), o.lm_iterations(1, F_STAGE1)
    assert s1g.successful_steps == s1o.successful_steps == 1
    assert abs(s1g.final_cost - s1o.final_cost) <= 1e-9 * s1o.final_cost
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-9
    for a, b in zip(g.get_knots()[:2], o.get_knots()[:2]):
        assert rel(a, b) < 1e-9
    sg, so = g.optimize(50, F_STAGE1), o.optimize(50, F_STAGE1)
    assert sg.iterations == so.iterations and sg.termination == so.termination and sg.successful_steps == so.successful_steps
    assert abs(sg.final_cost - so.final_cost) <= 1e-9 * so.final_cost
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8                          # north-star bar: 1e-4
    assert abs(sg.mean_reproj_error - so.mean_reproj_error) < 1e-9


def test_config3_whole_sequence_both_stages_against_oracle(oracle_factory, gpu_factory):
    from helpers import F_STAGE2
    ds = syn.make_dataset(syn.CONFIGS[3])
    g = gpu_factory(); capi.load_dataset(g, ds)
    o = oracle_factory(); capi.load_dataset(o, ds)
    assert g.num_residuals()[0] == 2 * 1000 * 96
    sg, so = g.optimize(50, F_STAGE1), o.optimize(50, F_STAGE1)
    assert sg.iterations == so.iterations and sg.termination == so.termination
    assert abs(sg.final_cost - so.final_cost) <= 1e-9 * so.final_cost
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8
    s2g, s2o = g.optimize(10, F_STAGE2), o.optimize(10, F_STAGE2)
    assert s2g.iterations == s2o.iterations and s2g.num_tangent == 1
    assert abs(g.get_line_delay() - o.get_line_delay()) <= 1e-7 * abs(o.get_line_delay())
    # (with the reference's function_tolerance = 1e-4 the one-parameter stage stops where the oracle stops, not at the truth)
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8
