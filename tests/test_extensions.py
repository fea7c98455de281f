"""North-star extension flags CAM_INTRINSICS / TIME_OFFSET (the reference keeps both quantities fixed: SURVEY.md "Read this
first" #3 — with the bits clear they are pass-through, which every other test exercises).
CPU: the oracle's autodiff columns for the two new blocks against finite differences obtained by actually changing the
inputs (intrinsics passed to set_camera / the IMU->camera time offset).  GPU: analytic columns == oracle, LM parity."""
import numpy as np
import pytest

from helpers import F_STAGE1, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_scaled_parity

F_CI, F_TO = capi.FLAG_CAM_INTRINSICS, capi.FLAG_TIME_OFFSET


def _load(api, ds, intr=None, toff=None):
    W, H = ds["image_size"]
    api.set_camera(ds["model"], ds["intrinsics"] if intr is None else intr, W, H); api.set_board_points(ds["board_xyzw"])
    api.set_frames(ds["frame_t"], ds["corner_offsets"], ds["point_ids"], ds["uv"], ds["q_wc"], ds["p_wc"]); api.set_imu(ds["imu_t"], ds["accel"], ds["gyro"])
    api.batch_init_spline(ds["T_i_c_init"], ds["dt_so3_s"], ds["dt_r3_s"], ds["std_so3"], ds["std_r3"],
                          ds["time_offset_imu_to_cam_s"] if toff is None else toff, ds["init_line_delay_s"], acc_bias=ds["acc_bias"], gyr_bias=ds["gyr_bias"],
                          dispatch_fov=ds["model"] == cm.FOV)
    api.set_known_gravity_dir(ds["gravity"])


@pytest.mark.parametrize("k", range(7))
def test_oracle_intrinsics_gradient_fd(oracle_factory, k):
    cfg = syn.config5(k); cfg.n_frames = 10
    ds = syn.make_dataset(cfg)
    o = oracle_factory(2); _load(o, ds)
    n = o.num_tangent(F_CI)
    K = len(ds["intrinsics"])
    assert n == K
    g = o.evaluate(F_CI)[2]
    for i in range(K):
        h = 1e-6 * abs(ds["intrinsics"][i]) if abs(ds["intrinsics"][i]) > 1e-12 else 1e-6
        kp, km = np.array(ds["intrinsics"], dtype=float), np.array(ds["intrinsics"], dtype=float)
        kp[i] += h; km[i] -= h
        op, om = oracle_factory(2), oracle_factory(2)
        _load(op, ds, intr=kp); _load(om, ds, intr=km)
        cp, cm_ = op.evaluate(0, gradient=False, residuals=False)[0], om.evaluate(0, gradient=False, residuals=False)[0]
        fd = (cp - cm_) / (2 * h)
        assert abs(fd - g[i]) <= 1e-5 * max(abs(fd), abs(g[i])) + 1e-10 * cp / h, (i, fd, g[i])     # second term: round-off of the difference


def test_oracle_time_offset_gradient_fd(oracle_factory):
    ds = syn.make_dataset(syn.tiny_config(n_frames=30, imu_rate_hz=200.0, seed=4))
    base = ds["time_offset_imu_to_cam_s"] + 1.2345e-3      # keeps every IMU stamp away from the [t0, tend) window edges
    o = oracle_factory(2); _load(o, ds, toff=base)
    assert o.num_tangent(F_TO) == 1
    g = o.evaluate(F_TO)[2][0]
    h = 1e-6
    op, om = oracle_factory(2), oracle_factory(2)
    _load(op, ds, toff=base + h); _load(om, ds, toff=base - h)
    assert op.num_residuals() == om.num_residuals()
    fd = (op.evaluate(0, gradient=False, residuals=False)[0] - om.evaluate(0, gradient=False, residuals=False)[0]) / (2 * h)
    assert abs(fd - g) <= 1e-4 * abs(fd), (fd, g)


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(8))
def test_gpu_extension_columns_match_oracle(oracle_factory, gpu_factory, k):
    cfg = syn.config5(k); cfg.n_frames = 16
    ds = syn.make_dataset(cfg)
    o = oracle_factory(); _load(o, ds)
    g = gpu_factory(); _load(g, ds)
    for flags in (F_CI, F_TO, F_STAGE1 | F_CI | F_TO, F_STAGE1 | F_CI | F_TO | capi.FLAG_IMU_BIASES | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_GRAVITY_DIR | capi.FLAG_IMU_INTRINSICS):
        assert o.num_tangent(flags) == g.num_tangent(flags)
        co, ro, go, Ho = o.evaluate(flags, hessian=True)
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        assert abs(cg - co) <= 1e-9 * co and rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9 and rel(Hg, Ho) < 1e-9
        assert_scaled_parity(g, flags, (co, ro, go, Ho), (cg, rg, gg, Hg))


@pytest.mark.gpu
def test_gpu_extension_lm_and_pass_through(oracle_factory, gpu_factory):
    ds = dict(syn.make_dataset(syn.tiny_config(cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), n_frames=50, imu_rate_hz=200.0, seed=31)))
    o = oracle_factory(); g = gpu_factory()
    # pass-through with the bits clear: intrinsics and time offset come back exactly as given (reference behaviour)
    _load(g, ds)
    g.optimize(5, F_STAGE1)
    assert np.array_equal(g.get_camera_intrinsics(7), np.asarray(ds["intrinsics"], dtype=float))
    assert g.get_time_offset() == ds["time_offset_imu_to_cam_s"]
    # start 2 ms off in time offset and 1 % off in focal length; free both
    k0 = np.array(ds["intrinsics"], dtype=float); k0[0] *= 1.01
    t0 = ds["time_offset_imu_to_cam_s"] + 2e-3
    _load(o, ds, intr=k0, toff=t0); g2 = gpu_factory(); _load(g2, ds, intr=k0, toff=t0)
    flags = F_STAGE1 | F_CI | F_TO
    so, sg = o.optimize(30, flags), g2.optimize(30, flags)
    assert sg.iterations == so.iterations
    assert rel(g2.get_camera_intrinsics(7), o.get_camera_intrinsics(7)) < 1e-7 and abs(g2.get_time_offset() - o.get_time_offset()) < 1e-9
    assert sg.final_cost < 0.5 * sg.initial_cost and abs(sg.final_cost - so.final_cost) <= 1e-7 * so.final_cost
    assert abs(g2.get_time_offset() - ds["time_offset_imu_to_cam_s"]) < 5e-4          # the 2 ms time-offset error is pulled back (s)
