"""The GPU's normal equations, gradient and residuals against the oracle entry by entry, each at its own scale (scaled_parity.py), on
the column sets, camera models, multi-chunk runs, bias priors and failed projections whose weak blocks the max-normalised comparison
cannot see: the bias, IMU-intrinsic and time-offset columns of imu_kernel, the rows of icc_bias_prior.cu, the gravity column and the
border branch of tile_flush in the persistent kernel, and the end knots of both splines."""
import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import SENTINEL, assert_scaled_parity
from test_gpu_bias_random_walk import WALK, _pair as _bias_pair, _perturb
from test_gpu_tmem_runs import _irregular_stamps_dataset, _ragged_dataset, checked_schedule, tmem_runs  # noqa: F401  (fixture)
from test_scaled_parity_metric import COLUMN_SETS, config5_dataset, load_with_imu_intrinsics

pytestmark = pytest.mark.gpu
F_GRAV1 = F_STAGE1 | capi.FLAG_GRAVITY_DIR
F_BIAS = F_STAGE1 | capi.FLAG_IMU_BIASES


def _check(o, g, flags, extra_gpu_columns=0):
    """Cost to 1e-9 relative and everything else at its own scale; `extra_gpu_columns`: trailing intrinsic columns the oracle of
    that model does not have."""
    ev_o, ev_g = o.evaluate(flags, hessian=True), g.evaluate(flags, hessian=True)
    assert abs(ev_g[0] - ev_o[0]) <= 1e-9 * abs(ev_o[0])
    if extra_gpu_columns:
        m = len(ev_o[2])
        assert len(ev_g[2]) == m + extra_gpu_columns
        ev_g = (ev_g[0], ev_g[1], ev_g[2][:m], np.ascontiguousarray(ev_g[3][:m, :m]))
    return assert_scaled_parity(o, flags, ev_o, ev_g)


@pytest.mark.parametrize("k", range(8))
def test_config5_every_column_set(oracle_factory, gpu_factory, eval_path, k):
    ds = config5_dataset(k)
    o, g = oracle_factory(), gpu_factory()
    load_with_imu_intrinsics(o, ds); load_with_imu_intrinsics(g, ds)
    for flags in COLUMN_SETS:
        _check(o, g, flags)


def _other_models():
    from test_gpu_fisheye_radtan import K_SKEW as FR_SKEW, _pair as fr_pair, _tiny as fr_tiny
    from test_gpu_parity import _pair
    from test_gpu_rational import K_SKEW as RAT_SKEW, _pair as rat_pair, _tiny as rat_tiny
    from test_omni_radtan import K17, OMNI, omni_oracle
    from test_scaramuzza import K_FISH, SCARA, scara_oracle
    prt = syn.tiny_config(cm.PINHOLE_RADIAL_TANGENTIAL, (440.0, 1.01, 0.2, 480.0, 270.0, -0.1, 0.02, -0.003, 1e-3, -2e-3), seed=3)
    return {
        "pinhole_radtan": lambda of, gf: _pair(of, gf, syn.make_dataset(prt), known_gravity=False) + (0,),
        "omni_radtan": lambda of, gf: _pair(omni_oracle, gf, syn.make_dataset(syn.tiny_config(OMNI, tuple(K17), n_frames=20, seed=9)),
                                            known_gravity=False) + (0,),
        "scaramuzza": lambda of, gf: _pair(scara_oracle, gf, syn.make_dataset(syn.tiny_config(SCARA, tuple(K_FISH), n_frames=20, seed=9)),
                                           known_gravity=False) + (0,),
        "rational": lambda of, gf: rat_pair(gf, syn.make_dataset(rat_tiny(RAT_SKEW, n_frames=20, seed=11)), known_gravity=False) + (3,),
        "fisheye62": lambda of, gf: fr_pair(gf, syn.make_dataset(fr_tiny(FR_SKEW, n_frames=20, seed=11)), known_gravity=False) + (3,),
    }


@pytest.mark.parametrize("model", ["pinhole_radtan", "omni_radtan", "scaramuzza", "rational", "fisheye62"])
def test_other_camera_models_with_intrinsics(oracle_factory, gpu_factory, eval_path, model):
    """The rational and Fisheye62 oracles hold the last three intrinsics constant: their columns are checked against central
    differences in the models' own test files, the leading ones here."""
    o, g, extra = _other_models()[model](oracle_factory, gpu_factory)
    _check(o, g, F_ALL | capi.FLAG_CAM_INTRINSICS, extra)


@pytest.mark.parametrize("case", ["ragged", "stamps", "1khz"])
def test_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs, case):  # noqa: F811
    ds = {"ragged": _ragged_dataset, "stamps": _irregular_stamps_dataset,
          "1khz": lambda: syn.make_dataset(syn.tiny_config(n_frames=20, imu_rate_hz=1000.0))}[case]()
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    ref = {flags: o.evaluate(flags, hessian=True) for flags in (F_ALL, F_GRAV1)}
    seen = set()
    for cap in (1, 7, 13):
        tmem_runs(cap)
        g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
        feats = checked_schedule(g, ds, cap)
        seen |= feats["vision"] | feats["imu"]
        for flags, ev_o in ref.items():
            ev_g = g.evaluate(flags, hessian=True)
            assert abs(ev_g[0] - ev_o[0]) <= 1e-9 * ev_o[0]
            assert_scaled_parity(o, flags, ev_o, ev_g)
        g.close()
    assert {"carry", "straddle"} <= seen, seen


@pytest.mark.parametrize("sensors", list(WALK))
def test_bias_prior_many_knots(eval_path, sensors):
    """0.5 s bias knots on a 0.8 s sequence: every bias column is touched by prior rows and by few IMU rows."""
    g, o = _bias_pair(syn.make_dataset(syn.tiny_config(n_frames=24)), 0.5, WALK[sensors])
    _perturb(g, o)
    assert g.num_bias_prior_residuals() == o.num_bias_prior_residuals() > 0
    for flags in (F_BIAS, F_ALL):
        _check(o, g, flags)


def test_failed_projections(oracle_factory, gpu_factory, eval_path):
    """A board point behind the camera: 1e10 residuals with zero derivative in every frame, checked position for position, and the
    other residuals at their own scale."""
    cfg = syn.tiny_config(cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513), seed=5)
    ds = dict(syn.make_dataset(cfg))
    board = ds["board_xyzw"].copy(); board[3, :3] = [0.0, 0.0, 50.0]
    ds["board_xyzw"] = board
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
    for flags in (F_STAGE1, F_ALL):
        _check(o, g, flags)
    assert (g.evaluate(F_STAGE1, gradient=False)[1] == SENTINEL).sum() == 2 * len(ds["frame_t"])
