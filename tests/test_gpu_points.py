"""SplineOptimFlags::POINTS on the GPU (icc_points.cu) against the oracle: the board points as 4-vector parameter blocks with
ceres::HomogeneousVectorParameterization(4) (reference: SetFixedParams, core/spline_trajectory_estimator.impl.h:136-152).
  * cost, J^T r and J^T J (products with random vectors: point x point, point x knot, point x T_i_c blocks) at 1e-9,
  * J^T r against central differences of the GPU's own cost through the NumPy Plus,
  * one LM iteration and the whole run (iteration counts, cost, T_i_c, the optimised points),
  * the points survive a following run WITHOUT the flag in both state buffers,
  * border width: config 2's 96-point board (294 border columns) solves, config 4's 144-point board is refused with ICC_ERR_UNSUPPORTED."""
import numpy as np
import pytest

from helpers import F_STAGE1, TangentWalker, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_block_probes, probe_reference

pytestmark = pytest.mark.gpu
FLAGS = F_STAGE1 | capi.FLAG_POINTS

MODELS = [(cm.DIVISION_UNDISTORTION, (437.1, 1.0, 489.1, 270.9, -1.44e-6)), (cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513))]


def _pair(oracle_factory, gpu_factory, ds):
    g = gpu_factory(); capi.load_dataset(g, ds)
    o = oracle_factory(); capi.load_dataset(o, ds)
    return g, o


@pytest.mark.parametrize("model,intr", MODELS)
def test_points_jacobian_parity(oracle_factory, gpu_factory, eval_path, model, intr):
    ds = syn.make_dataset(syn.tiny_config(model=model, intr=intr, n_frames=16))
    g, o = _pair(oracle_factory, gpu_factory, ds)
    npts = len(ds["board_xyzw"])
    n = g.num_tangent(FLAGS)
    assert n == o.num_tangent(FLAGS) == g.num_tangent(F_STAGE1) + 3 * npts
    cg, rg, gg, _ = g.evaluate(FLAGS)
    co, ro, go, _ = o.evaluate(FLAGS)
    assert abs(cg - co) <= 1e-11 * co and rel(rg, ro) < 1e-9
    assert rel(gg, go) < 1e-9
    assert rel(gg[n - 3 * npts:], go[n - 3 * npts:]) < 1e-9          # the point block on its own
    rng = np.random.default_rng(8)
    V = rng.normal(size=(4, n)); V[1, : n - 3 * npts] = 0.0; V[2, n - 3 * npts:] = 0.0
    for a, b in zip(g.normal_matvec(FLAGS, V), o.normal_matvec(FLAGS, V)):
        assert rel(a, b) < 1e-9
    assert_block_probes(g, probe_reference(o, FLAGS, rng))


def test_points_gradient_against_finite_differences(gpu_factory):
    ds = syn.make_dataset(syn.tiny_config(n_frames=10))
    g = gpu_factory(); capi.load_dataset(g, ds)
    npts = len(ds["board_xyzw"]); n = g.num_tangent(FLAGS)
    _, _, grad, _ = g.evaluate(FLAGS)
    w = TangentWalker(g, FLAGS)
    rng = np.random.default_rng(5)
    for trial in range(3):
        d = np.zeros(n)
        if trial < 2: d[n - 3 * npts:] = rng.normal(size=3 * npts)
        else: d = rng.normal(size=n)
        eps = 1e-7
        fd = (w.cost(eps * d) - w.cost(-eps * d)) / (2 * eps)
        assert abs(fd - grad @ d) <= 2e-5 * max(abs(fd), abs(grad @ d)), (trial, fd, grad @ d)
    w.restore()


def test_points_lm_parity_and_state(oracle_factory, gpu_factory):
    ds = syn.make_dataset(syn.tiny_config(n_frames=24))
    rng = np.random.default_rng(3)
    ds["board_xyzw"] = ds["board_xyzw"].copy(); ds["board_xyzw"][:, :3] += 2e-3 * rng.normal(size=(len(ds["board_xyzw"]), 3))    # a board that is 2 mm off
    g, o = _pair(oracle_factory, gpu_factory, ds)
    s1g, s1o = g.lm_iterations(1, FLAGS), o.lm_iterations(1, FLAGS)
    assert s1g.successful_steps == s1o.successful_steps == 1
    assert abs(s1g.final_cost - s1o.final_cost) <= 1e-9 * s1o.final_cost
    assert rel(g.get_board_points(), o.get_board_points()) < 1e-9
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-9
    sg, so = g.optimize(30, FLAGS), o.optimize(30, FLAGS)
    assert sg.iterations == so.iterations and sg.termination == so.termination and sg.successful_steps == so.successful_steps
    assert abs(sg.final_cost - so.final_cost) <= 1e-8 * so.final_cost
    assert rel(g.get_board_points(), o.get_board_points()) < 1e-7
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-7
    pts = g.get_board_points()
    assert np.abs(pts - ds["board_xyzw"]).max() > 1e-5                 # the points moved
    assert np.allclose(np.linalg.norm(pts, axis=1), np.linalg.norm(ds["board_xyzw"], axis=1), rtol=1e-12)   # Plus keeps |x| (Householder)
    # a run without the flag keeps the optimised points constant in both state buffers
    s2g, s2o = g.optimize(5, F_STAGE1), o.optimize(5, F_STAGE1)
    assert s2g.iterations == s2o.iterations
    assert abs(s2g.final_cost - s2o.final_cost) <= 1e-8 * s2o.final_cost
    assert rel(g.get_board_points(), pts) == 0.0
    cg = g.evaluate(F_STAGE1, residuals=False, gradient=False)[0]; co = o.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    assert abs(cg - co) <= 1e-8 * co


def test_points_set_after_init_reaches_the_device(gpu_factory):
    ds = syn.make_dataset(syn.tiny_config(n_frames=10))
    g = gpu_factory(); capi.load_dataset(g, ds)
    c0 = g.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    p = ds["board_xyzw"].copy(); p[:, 0] += 1e-3
    g.set_board_points(p)
    c1 = g.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    assert c1 != c0
    g.set_board_points(2.0 * ds["board_xyzw"])                         # homogeneous scale: same points
    c2 = g.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    assert abs(c2 - c0) <= 1e-12 * c0


def test_points_wide_border(oracle_factory, gpu_factory):
    """The board-point columns sit in the border of the banded + bordered solver.  BASELINE config 2's 96-point board (294 border columns)
    solves; config 4's 144-point board (438) is beyond the solver's shared-memory window (the limit at kd = 35 is 133 points next to T_i_c)
    and is refused loudly with ICC_ERR_UNSUPPORTED -- evaluation (cost, J^T r, J^T J products) works at any width."""
    import dataclasses
    ds = syn.make_dataset(dataclasses.replace(syn.CONFIGS[2], n_frames=60))
    g, o = _pair(oracle_factory, gpu_factory, ds)
    assert len(ds["board_xyzw"]) == 96
    cg, _, gg, _ = g.evaluate(FLAGS, residuals=False)
    co, _, go, _ = o.evaluate(FLAGS, residuals=False)
    assert abs(cg - co) <= 1e-10 * co and rel(gg, go) < 1e-9
    sg, so = g.lm_iterations(2, FLAGS), o.lm_iterations(2, FLAGS)
    assert sg.successful_steps == so.successful_steps and sg.num_tangent == so.num_tangent
    assert abs(sg.final_cost - so.final_cost) <= 1e-8 * so.final_cost
    assert rel(g.get_board_points(), o.get_board_points()) < 1e-7

    ds = syn.make_dataset(dataclasses.replace(syn.CONFIGS[4], n_frames=40))
    g, o = _pair(oracle_factory, gpu_factory, ds)
    assert len(ds["board_xyzw"]) == 144
    cg, _, gg, _ = g.evaluate(FLAGS, residuals=False)
    co, _, go, _ = o.evaluate(FLAGS, residuals=False)
    assert abs(cg - co) <= 1e-10 * co and rel(gg, go) < 1e-9
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED"):
        g.lm_iterations(1, FLAGS)
    s = g.lm_iterations(1, F_STAGE1)                                   # the handle stays usable
    assert s.successful_steps == 1
