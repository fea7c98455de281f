"""Parity of the CUDA path (through the C-ABI) against the CPU oracle on identical seeded inputs.
FP64 tolerances: residuals / cost / J^T r / J^T J relative 1e-9 (observed ~1e-14), and 1e-9 again with every block at its own scale
(scaled_parity.py: Jacobi-scaled J^T J, J^T r against |r| sqrt(diag), residuals per kind; observed <= 4e-14 on an H100); LM end state relative 1e-8;
north-star bar on converged T_cam_imu / line delay: 1e-4 relative."""
import os

import numpy as np
import pytest

from golden_io import golden_files, load_golden
from helpers import F_ALL, F_STAGE1, F_STAGE2, TangentWalker, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_scaled_parity

pytestmark = pytest.mark.gpu
TOL = 1e-9


def _pair(oracle_factory, gpu_factory, ds, **kw):
    o = oracle_factory(); capi.load_dataset(o, ds, **kw)
    g = gpu_factory(); capi.load_dataset(g, ds, **kw)
    return o, g


def _assert_eval_parity(o, g, flags, hessian=True):
    co, ro, go, Ho = o.evaluate(flags, hessian=hessian)
    cg, rg, gg, Hg = g.evaluate(flags, hessian=hessian)
    assert abs(cg - co) <= TOL * abs(co)
    assert rel(rg, ro) < TOL and rel(gg, go) < TOL
    if hessian:
        assert rel(Hg, Ho) < TOL
        assert np.array_equal(Hg, Hg.T)
        assert_scaled_parity(g, flags, (co, ro, go, Ho), (cg, rg, gg, Hg))   # each block at its own scale
    c2 = g.evaluate(flags, residuals=False, gradient=False)[0]     # cost-only kernels agree with the Jacobian kernels
    assert abs(c2 - cg) <= 1e-12 * abs(cg)


@pytest.mark.parametrize("k", range(8))
def test_eval_parity_every_camera_model_all_blocks(oracle_factory, gpu_factory, k, eval_path):
    cfg = syn.config5(k); cfg.n_frames = 20
    o, g = _pair(oracle_factory, gpu_factory, syn.make_dataset(cfg), known_gravity=False)
    for flags in (F_STAGE1, F_ALL, F_STAGE2, capi.FLAG_T_I_C, capi.FLAG_SPLINE | capi.FLAG_GYR_BIAS, capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS,
                  F_STAGE1 | capi.FLAG_GRAVITY_DIR):   # stage 1 with unknown gravity: the gravity columns on the persistent IMU items
        _assert_eval_parity(o, g, flags)


def test_eval_parity_imu_intrinsics_flag(oracle_factory, gpu_factory):
    """SplineOptimFlags::IMU_INTRINSICS (SetFixedParams impl.h:166-178): misalignment + scale blocks of both triads, with
    non-trivial intrinsics so that every derivative is exercised."""
    ds = syn.make_dataset(syn.tiny_config(seed=13))
    acc_i = (0.01, -0.02, 0.015, 1.02, 0.98, 1.01); gyr_i = (0.01, -0.005, 0.02, -0.015, 0.008, 0.012, 0.99, 1.03, 1.01)
    def load(api):
        W, H = ds["image_size"]
        api.set_camera(ds["model"], ds["intrinsics"], W, H); api.set_board_points(ds["board_xyzw"])
        api.set_frames(ds["frame_t"], ds["corner_offsets"], ds["point_ids"], ds["uv"], ds["q_wc"], ds["p_wc"]); api.set_imu(ds["imu_t"], ds["accel"], ds["gyro"])
        api.batch_init_spline(ds["T_i_c_init"], ds["dt_so3_s"], ds["dt_r3_s"], ds["std_so3"], ds["std_r3"], ds["time_offset_imu_to_cam_s"], ds["init_line_delay_s"],
                              acc_intrinsics=acc_i, gyr_intrinsics=gyr_i, acc_bias=ds["acc_bias"], gyr_bias=ds["gyr_bias"])
    o = oracle_factory(); load(o)
    g = gpu_factory(); load(g)
    for flags in (capi.FLAG_IMU_INTRINSICS, F_ALL | capi.FLAG_IMU_INTRINSICS, F_STAGE1 | capi.FLAG_IMU_INTRINSICS):
        assert o.num_tangent(flags) == g.num_tangent(flags)
        _assert_eval_parity(o, g, flags)
    so, sg = o.optimize(20, F_STAGE1 | capi.FLAG_IMU_INTRINSICS | capi.FLAG_IMU_BIASES), g.optimize(20, F_STAGE1 | capi.FLAG_IMU_INTRINSICS | capi.FLAG_IMU_BIASES)
    assert sg.iterations == so.iterations and abs(sg.final_cost - so.final_cost) <= 1e-7 * so.final_cost


def test_eval_parity_pinhole_radial_tangential(oracle_factory, gpu_factory, eval_path):
    cfg = syn.tiny_config(cm.PINHOLE_RADIAL_TANGENTIAL, (440.0, 1.01, 0.2, 480.0, 270.0, -0.1, 0.02, -0.003, 1e-3, -2e-3), seed=3)
    o, g = _pair(oracle_factory, gpu_factory, syn.make_dataset(cfg), known_gravity=False)
    _assert_eval_parity(o, g, F_ALL)


def test_eval_parity_uneven_knot_spacing(oracle_factory, gpu_factory, eval_path):
    """dt_so3 != dt_r3: different segment indices per spline, wider band, IMU cells cut at both knot grids."""
    for a, b in ((0.04, 0.07), (0.09, 0.05)):
        o, g = _pair(oracle_factory, gpu_factory, syn.make_dataset(syn.tiny_config(dt_so3_s=a, dt_r3_s=b, n_frames=30)), known_gravity=False)
        _assert_eval_parity(o, g, F_ALL)


@pytest.mark.parametrize("path", golden_files(), ids=[os.path.basename(p) for p in golden_files()])
def test_gpu_matches_committed_golden(gpu_factory, path, eval_path):
    ds = load_golden(path)
    g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
    for tag, flags in (("stage1", F_STAGE1), ("all", F_ALL), ("stage2", F_STAGE2)):
        c, r, gr, H = g.evaluate(flags, hessian=True)
        assert abs(c - float(ds[f"{tag}_cost"])) <= TOL * abs(c)
        assert rel(r, ds[f"{tag}_residuals"]) < TOL and rel(gr, ds[f"{tag}_gradient"]) < TOL and rel(H, ds[f"{tag}_hessian"]) < TOL
        golden = tuple(ds[f"{tag}_{x}"] for x in ("cost", "residuals", "gradient", "hessian"))
        assert_scaled_parity(g, flags, golden, (c, r, gr, H))
    g2 = gpu_factory(); capi.load_dataset(g2, ds, known_gravity=True)
    s1 = g2.optimize(50, F_STAGE1)
    assert s1.iterations == int(ds["lm_stage1_iterations"]) and s1.gpu_launches > 0
    assert rel(g2.get_T_i_c(), ds["lm_stage1_T_i_c"]) < 1e-8
    assert abs(s1.mean_reproj_error - float(ds["lm_stage1_reproj"])) < 1e-8
    s2 = g2.optimize(10, F_STAGE2)
    assert s2.iterations == int(ds["lm_stage2_iterations"])
    assert abs(g2.get_line_delay() - float(ds["lm_stage2_line_delay"])) <= 1e-8 * abs(float(ds["lm_stage2_line_delay"]))


def test_ragged_and_empty_frames(oracle_factory, gpu_factory, eval_path):
    """Frames with 0, 1, 33 and all corners, shuffled point ids, a frame outside the IMU range."""
    ds = dict(syn.make_dataset(syn.tiny_config(grid=(9, 5), n_frames=16)))
    C = 45
    keep_counts = [0, 1, 33, 45, 7, 32, 31, 45, 2, 45, 45, 40, 45, 45, 3, 45]
    rng = np.random.default_rng(0)
    off, ids, uv = [0], [], []
    for f, n in enumerate(keep_counts):
        sel = np.sort(rng.choice(C, size=n, replace=False))
        ids.append(ds["point_ids"][f * C + sel]); uv.append(ds["uv"][f * C + sel]); off.append(off[-1] + n)
    ds["corner_offsets"] = np.array(off, dtype=np.int32); ds["point_ids"] = np.concatenate(ids).astype(np.int32); ds["uv"] = np.concatenate(uv)
    o, g = _pair(oracle_factory, gpu_factory, ds, known_gravity=False)
    assert o.num_residuals() == g.num_residuals() and g.num_residuals()[0] == 2 * sum(keep_counts)
    _assert_eval_parity(o, g, F_ALL)


def test_failed_projections_give_constant_1e10_residuals(oracle_factory, gpu_factory, eval_path):
    """SURVEY quirk q12: a point outside the unified model's domain => residual (1e10, 1e10) with zero derivative."""
    cfg = syn.tiny_config(cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513), seed=5)
    ds = dict(syn.make_dataset(cfg))
    board = ds["board_xyzw"].copy(); board[3, :3] = [0.0, 0.0, 50.0]       # far behind the camera
    ds["board_xyzw"] = board
    o, g = _pair(oracle_factory, gpu_factory, ds)
    co, ro, go, _ = o.evaluate(F_STAGE1)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    assert (ro == 1e10).sum() == (rg == 1e10).sum() == 2 * len(ds["frame_t"])
    assert np.array_equal(ro == 1e10, rg == 1e10)
    assert abs(cg - co) <= 1e-12 * co and rel(gg, go) < TOL


def test_fov_reference_quirk_and_extension(oracle_factory, gpu_factory):
    cfg = syn.config5(5); cfg.n_frames = 10
    ds = syn.make_dataset(cfg)
    o = oracle_factory(); capi.load_dataset(o, ds, dispatch_fov=False)
    g = gpu_factory(); capi.load_dataset(g, ds, dispatch_fov=False)
    ro = o.evaluate(F_STAGE1)[1]; rg = g.evaluate(F_STAGE1)[1]
    nv = g.num_residuals()[0]
    assert np.all(rg[:nv] == 1e10) and np.all(ro[:nv] == 1e10)          # reference: FOV is never dispatched


def test_global_shutter_path(oracle_factory, gpu_factory):
    ds = dict(syn.make_dataset(syn.tiny_config())); ds["init_line_delay_s"] = 0.0
    o, g = _pair(oracle_factory, gpu_factory, ds)
    assert g.num_residuals() == o.num_residuals() and g.num_residuals()[0] == 0
    _assert_eval_parity(o, g, F_STAGE1)
    assert abs(g.mean_reprojection_error() - o.mean_reprojection_error()) < 1e-9


def test_no_imu_and_imu_only_slices(oracle_factory, gpu_factory, eval_path):
    ds = dict(syn.make_dataset(syn.tiny_config()))
    ds["imu_t"] = ds["imu_t"][:0]; ds["accel"] = ds["accel"][:0]; ds["gyro"] = ds["gyro"][:0]
    o, g = _pair(oracle_factory, gpu_factory, ds)
    assert g.num_residuals()[1:] == (0, 0)
    _assert_eval_parity(o, g, F_STAGE1)


def test_gradient_matches_finite_differences_of_gpu_cost(gpu_factory, eval_path):
    ds = syn.make_dataset(syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), seed=9))
    g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
    flags = F_STAGE1 | capi.FLAG_GRAVITY_DIR | capi.FLAG_IMU_BIASES
    grad = g.evaluate(flags)[2]
    w = TangentWalker(g, flags)
    rng = np.random.default_rng(1)
    for _ in range(3):
        d = rng.normal(size=w.n); eps = 1e-7
        fd = (w.cost(eps * d) - w.cost(-eps * d)) / (2 * eps)
        assert abs(fd - grad @ d) <= 2e-6 * abs(fd)


def test_trajectory_getters(oracle_factory, gpu_factory):
    ds = syn.make_dataset(syn.tiny_config())
    o, g = _pair(oracle_factory, gpu_factory, ds)
    t_used = g.imu_used()[0]
    t_ns = np.concatenate([(t_used * 1e9).astype(np.int64), np.array([-5, int(1e12)], dtype=np.int64)])   # incl. out-of-range stamps
    a, b = g.eval_trajectory(t_ns), o.eval_trajectory(t_ns)
    assert np.array_equal(a["valid"], b["valid"]) and a["valid"][-1] == 0 and a["valid"][-2] == 0
    for key in ("gyro", "accel", "gyro_bias", "accel_bias", "pose_q", "pose_p"):
        assert rel(a[key], b[key]) < TOL, key


def test_imu_stamps_on_knot_boundaries_and_repeated(oracle_factory, gpu_factory, eval_path):
    """IMU stamps that fall exactly on knot-interval boundaries, repeated stamps and an irregular rate: the cells of the sorted stream are
    found by bisection for the next boundary (icc_api.cu: cells_by_bisection) and the relative integer times are derived on the device
    (imu_times_kernel); both must reproduce CalcTimes sample by sample.  The same samples shuffled take the general (sequential) path."""
    ds = dict(syn.make_dataset(syn.tiny_config(n_frames=30, dt_so3_s=0.04, dt_r3_s=0.07)))
    rng = np.random.default_rng(12)
    t0 = float(ds["frame_t"][0]) - ds["time_offset_imu_to_cam_s"]
    n = len(ds["imu_t"])
    t = np.sort(rng.uniform(ds["imu_t"][0], ds["imu_t"][-1], size=n))
    k = np.arange(0, n, 7)
    t[k] = t0 + 0.04 * np.round((t[k] - t0) / 0.04)                     # on SO(3) knot boundaries (as exactly as a double allows)
    k = np.arange(3, n, 11)
    t[k] = t0 + 0.07 * np.round((t[k] - t0) / 0.07)                     # on R^3 knot boundaries
    t = np.sort(t); t[5::13] = t[4::13][: len(t[5::13])]                # repeated stamps
    t = np.sort(t)
    ds["imu_t"] = t
    g = gpu_factory(); capi.load_dataset(g, ds)
    o = oracle_factory(); capi.load_dataset(o, ds)
    assert g.num_residuals() == o.num_residuals()
    for a, b in zip(g.imu_used(), o.imu_used()):
        assert np.array_equal(a, b)
    cg, rg, gg, _ = g.evaluate(F_STAGE1)
    co, ro, go, _ = o.evaluate(F_STAGE1)
    assert abs(cg - co) <= 1e-10 * co and rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9
    perm = rng.permutation(n)
    dsh = dict(ds); dsh["imu_t"], dsh["accel"], dsh["gyro"] = t[perm], ds["accel"][perm], ds["gyro"][perm]
    s = gpu_factory(); capi.load_dataset(s, dsh)
    cs = s.evaluate(F_STAGE1, residuals=False, gradient=False)[0]
    assert s.num_residuals() == g.num_residuals() and abs(cs - cg) <= 1e-12 * cg
