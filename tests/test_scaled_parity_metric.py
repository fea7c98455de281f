"""The scale-aware comparison (scaled_parity.py) and the oracle it holds the GPU to, on the CPU:
  * it rejects perturbations of one block, one gradient entry and one residual next to a 1e10 sentinel that helpers.rel passes, and
    names the block;
  * it is invariant under column scaling;
  * the oracle's J^T J and J^T r equal J^T J and J^T r of its own dense Jacobian accumulated in extended precision, Jacobi-scaled, far
    below the 1e-9 the GPU is held to (measured: 7.4e-16), for every config-5 camera model and the column sets of the GPU tests;
  * the oracle's Jacobian columns equal central differences of its residuals, in every column block."""
import ctypes

import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, TangentWalker, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import (SENTINEL, TOL, assert_gradient, assert_hessian, assert_residuals, column_blocks, gradient_errors,
                           hessian_errors, residual_kinds, residual_norm)

F_WIDE = F_ALL | capi.FLAG_IMU_INTRINSICS | capi.FLAG_CAM_INTRINSICS | capi.FLAG_TIME_OFFSET
COLUMN_SETS = (F_STAGE1, F_STAGE1 | capi.FLAG_GRAVITY_DIR, F_ALL, F_STAGE2, capi.FLAG_T_I_C, capi.FLAG_SPLINE | capi.FLAG_GYR_BIAS,
               capi.FLAG_GRAVITY_DIR | capi.FLAG_ACC_BIAS, F_ALL | capi.FLAG_IMU_INTRINSICS,
               F_ALL | capi.FLAG_CAM_INTRINSICS | capi.FLAG_TIME_OFFSET)
ACC_I = (0.01, -0.02, 0.015, 1.02, 0.98, 1.01)                                   # non-trivial IMU intrinsics: every derivative is exercised
GYR_I = (0.01, -0.005, 0.02, -0.015, 0.008, 0.012, 0.99, 1.03, 1.01)
DP = ctypes.POINTER(ctypes.c_double)


def config5_dataset(k):
    cfg = syn.config5(k); cfg.n_frames = 20
    return syn.make_dataset(cfg)


def load_with_imu_intrinsics(api, ds, intrinsics=None, time_offset=None, acc_i=ACC_I, gyr_i=GYR_I):
    """load_dataset with unknown gravity and non-trivial IMU intrinsics (optionally other camera intrinsics or time offset)."""
    W, H = ds["image_size"]
    api.set_camera(ds["model"], ds["intrinsics"] if intrinsics is None else intrinsics, W, H); api.set_board_points(ds["board_xyzw"])
    api.set_frames(ds["frame_t"], ds["corner_offsets"], ds["point_ids"], ds["uv"], ds["q_wc"], ds["p_wc"])
    api.set_imu(ds["imu_t"], ds["accel"], ds["gyro"])
    api.batch_init_spline(ds["T_i_c_init"], ds["dt_so3_s"], ds["dt_r3_s"], ds["std_so3"], ds["std_r3"],
                          ds["time_offset_imu_to_cam_s"] if time_offset is None else time_offset, ds["init_line_delay_s"],
                          acc_intrinsics=acc_i, gyr_intrinsics=gyr_i, acc_bias=ds["acc_bias"], gyr_bias=ds["gyr_bias"],
                          dispatch_fov=ds["model"] == cm.FOV)


def jacobian_dense(o, flags):
    J = np.zeros((sum(o.num_residuals()), o.num_tangent(flags)))
    o._call("jacobian_dense", [ctypes.c_int, DP], int(flags), J.ctypes.data_as(DP))
    return J


@pytest.fixture(scope="module")
def oracle3(oracle_factory):
    o = oracle_factory(); load_with_imu_intrinsics(o, config5_dataset(3))
    c, r, g, H = o.evaluate(F_ALL, hessian=True)
    return o, c, r, g, H


def _block(blocks, name):
    return next(b for b in blocks if b.name == name)


# ---- the metric sees what rel misses ------------------------------------------------------------------------------------------------
def test_hessian_block_perturbation_is_named(oracle3):
    o, _, _, _, H = oracle3
    blocks = column_blocks(o, F_ALL)
    ab, gr = _block(blocks, "acc_bias"), _block(blocks, "gravity")
    Hp = H.copy()
    Hp[ab.start:ab.stop, gr.start:gr.stop] *= 1.0 + 1e-6
    Hp[gr.start:gr.stop, ab.start:ab.stop] *= 1.0 + 1e-6
    assert rel(Hp, H) < TOL
    with pytest.raises(AssertionError, match=r"gravity\.[xyz] x acc_bias\[\d\]\.[xyz]"):
        assert_hessian(Hp, H, blocks)
    assert_hessian(H.copy(), H, blocks)


def test_hessian_structural_zero_is_checked(oracle3):
    o, _, _, _, H = oracle3
    blocks = column_blocks(o, F_ALL)
    i, j = _block(blocks, "T_i_c").start + 2, _block(blocks, "gravity").start + 1
    assert H[i, j] == 0.0                                                   # T_i_c only enters vision rows, gravity only IMU rows
    Hp = H.copy()
    Hp[i, j] = Hp[j, i] = 1e-6 * np.sqrt(H[i, i] * H[j, j])
    assert rel(Hp, H) < TOL
    with pytest.raises(AssertionError, match=r"T_i_c\.tz x gravity\.y"):
        assert_hessian(Hp, H, blocks)
    # a column whose oracle diagonal is zero must be exactly zero
    Hz, Hq = H.copy(), H.copy()
    Hz[:, i] = Hz[i, :] = 0.0
    Hq[:, i] = Hq[i, :] = 0.0; Hq[i, j] = Hq[j, i] = 1e-300
    assert np.isinf(hessian_errors(Hq, Hz)[i, j])


def test_gradient_entry_perturbation_is_named(oracle3):
    o, c, r, g, H = oracle3
    blocks = column_blocks(o, F_ALL)
    i = _block(blocks, "acc_bias").start + 4
    d, rn = np.diag(H), residual_norm(r)
    assert abs(rn * rn - 2 * c) <= 1e-12 * 2 * c                           # cost = |r|^2 / 2
    gp = g.copy(); gp[i] += 1e-6 * rn * np.sqrt(d[i])
    assert rel(gp, g) < TOL
    with pytest.raises(AssertionError, match=r"acc_bias\[1\]\.y"):
        assert_gradient(gp, g, d, rn, blocks)
    assert_gradient(g.copy(), g, d, rn, blocks)


def test_residual_next_to_a_sentinel_is_checked(oracle_factory):
    cfg = syn.tiny_config(cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513), seed=5)
    ds = dict(syn.make_dataset(cfg))
    board = ds["board_xyzw"].copy(); board[3, :3] = [0.0, 0.0, 50.0]              # far behind the camera: a failed projection per frame
    ds["board_xyzw"] = board
    o = oracle_factory(); capi.load_dataset(o, ds)
    _, r, _, _ = o.evaluate(F_STAGE1, gradient=False)
    kinds = residual_kinds(o, len(r))
    s = np.flatnonzero(r == SENTINEL)
    assert len(s) == 2 * len(ds["frame_t"])
    k = s[-1] + 1                                                           # the residual right after a sentinel pair
    assert r[k] != SENTINEL
    rp = r.copy(); rp[k] += 1e-6 * np.abs(r[r != SENTINEL][: kinds[0][2]]).max()
    assert rel(rp, r) < TOL
    with pytest.raises(AssertionError, match="vision"):
        assert_residuals(rp, r, kinds)
    rs = r.copy(); rs[s[0]] = SENTINEL * (1 + 1e-15)                         # a sentinel must be exact
    with pytest.raises(AssertionError, match="sentinel"):
        assert_residuals(rs, r, kinds)
    assert_residuals(r.copy(), r, kinds)


def test_metric_is_invariant_under_column_scaling(oracle3):
    o, c, r, g, H = oracle3
    rng = np.random.default_rng(7)
    n = H.shape[0]
    Hp = H + 1e-10 * np.sqrt(np.outer(np.diag(H), np.diag(H))) * rng.normal(size=(n, n)); Hp = 0.5 * (Hp + Hp.T)
    gp = g + 1e-10 * residual_norm(r) * np.sqrt(np.diag(H)) * rng.normal(size=n)
    S = 2.0 ** rng.integers(-20, 21, size=n)                                 # powers of two: the scaling itself is exact
    E0 = hessian_errors(Hp, H)
    E1 = hessian_errors(S[:, None] * Hp * S[None, :], S[:, None] * H * S[None, :])
    assert np.array_equal(E1, E0)
    e0 = gradient_errors(gp, g, np.diag(H), residual_norm(r))
    e1 = gradient_errors(S * gp, S * g, S * S * np.diag(H), residual_norm(r))
    assert np.array_equal(e1, e0)
    assert E0.max() > 1e-11 and e0.max() > 1e-11


# ---- the oracle is a sound reference at this scale ------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(8))
def test_oracle_normal_equations_match_extended_precision(oracle_factory, k):
    """J^T J and J^T r of the oracle's dense Jacobian in long double (one Jacobian of the widest column set; the columns of a block
    do not depend on which other blocks are free) against the oracle's own accumulation under every column set."""
    o = oracle_factory(); load_with_imu_intrinsics(o, config5_dataset(k))
    _, r, _, _ = o.evaluate(F_WIDE, gradient=False)
    J = jacobian_dense(o, F_WIDE).astype(np.longdouble)
    Hl, gl = J.T @ J, J.T @ r.astype(np.longdouble)
    wide = {b.name: b for b in column_blocks(o, F_WIDE)}
    worst = 0.0
    for flags in COLUMN_SETS:
        _, _, g, H = o.evaluate(flags, hessian=True)
        blocks = column_blocks(o, flags)
        cols = np.concatenate([np.arange(wide[b.name].start, wide[b.name].stop) for b in blocks])
        Hw, gw = Hl[np.ix_(cols, cols)].astype(np.float64), gl[cols].astype(np.float64)
        worst = max(worst, assert_hessian(H, Hw, blocks, tol=1e-13, what=f"oracle J^T J under flags {flags}"))
        worst = max(worst, assert_gradient(g, gw, np.diag(Hw), residual_norm(r), blocks, tol=1e-13))
    print(f"config5({k}): oracle against long double, Jacobi-scaled: {worst:.1e}")


def _fd_state(o, ds, flags):
    """Central-difference probes of one column: a function of a step along tangent column j -> residuals.  Spline, T_i_c, gravity,
    line delay and biases through TangentWalker; intrinsics and time offset by reloading a second oracle with the changed value
    and the first one's state."""
    w = TangentWalker(o, flags & ~(capi.FLAG_IMU_INTRINSICS | capi.FLAG_CAM_INTRINSICS | capi.FLAG_TIME_OFFSET))   # (their columns come last)
    blocks = {b.name: b for b in column_blocks(o, flags)}
    K = np.asarray(ds["intrinsics"], dtype=np.float64)

    def residuals(j, h):
        name = next(nm for nm, b in blocks.items() if b.start <= j < b.stop)
        if name in ("acc_intrinsics", "gyr_intrinsics", "cam_intrinsics", "time_offset"):
            q = j - blocks[name].start
            from oracle_api import new_oracle
            p = new_oracle()
            acc, gyr, intr, toff = np.array(ACC_I), np.array(GYR_I), K.copy(), ds["time_offset_imu_to_cam_s"]
            if name == "acc_intrinsics":
                acc[q] += h
            elif name == "gyr_intrinsics":
                gyr[q] += h
            elif name == "cam_intrinsics":
                intr[q] += h
            else:
                toff += h
            load_with_imu_intrinsics(p, ds, intrinsics=intr, time_offset=toff, acc_i=acc, gyr_i=gyr)
            so3, r3, ba, bg = o.get_knots()
            p.set_knots(so3, r3, ba, bg); p.set_T_i_c(o.get_T_i_c()); p.set_line_delay(o.get_line_delay()); p.set_known_gravity_dir(o.get_gravity())
            assert p.num_residuals() == o.num_residuals()
            return p.evaluate(0, gradient=False)[1]
        d = np.zeros(w.n); d[j] = h
        w.apply(d)
        try:
            return o.evaluate(flags, gradient=False)[1]
        finally:
            w.restore()
    return residuals


def test_oracle_jacobian_columns_match_central_differences(oracle_factory):
    """At least one column of every block, the first and last knots of each spline included; the step is set per column so that it
    changes the residuals by about 1e-4 of their norm, the comparison is at that column's norm."""
    ds = dict(syn.make_dataset(syn.tiny_config(n_frames=20, seed=13)))
    ds["time_offset_imu_to_cam_s"] = ds["time_offset_imu_to_cam_s"] + 1.2345e-3    # keeps every IMU stamp away from the window edges
    o = oracle_factory(); load_with_imu_intrinsics(o, ds)
    rng = np.random.default_rng(2)
    so3, r3, ba, bg = o.get_knots()
    o.set_knots(ba=ba + rng.normal(0, 0.02, ba.shape), bg=bg + rng.normal(0, 2e-3, bg.shape))
    flags = F_WIDE
    J = jacobian_dense(o, flags)
    _, r, _, _ = o.evaluate(flags, gradient=False)
    blocks = column_blocks(o, flags)
    assert [b.name for b in blocks] == ["so3", "r3", "T_i_c", "gravity", "line_delay", "acc_bias", "gyr_bias", "acc_intrinsics",
                                        "gyr_intrinsics", "cam_intrinsics", "time_offset"]
    cols = []
    for b in blocks:
        picks = {0, b.size - 1, int(rng.integers(b.size))}
        cols += [b.start + q for q in sorted(picks)]
    res = _fd_state(o, ds, flags)
    rn = np.linalg.norm(r)
    worst = {}
    for j in cols:
        cn = np.linalg.norm(J[:, j])
        assert cn > 0.0, j
        b = next(b for b in blocks if b.start <= j < b.stop)
        # the spline's time axis is integer nanoseconds, so a time-offset step of h s is rounded by up to 1 ns: 1e-4 s balances
        # that against the truncation error (measured 4.4e-6 here; 1.5e-5 at 1e-5 s, 7e-5 at 1e-6 s)
        h, tol = (1e-4, 1e-5) if b.name == "time_offset" else (1e-4 * rn / cn, 1e-6)
        fd = (res(j, h) - res(j, -h)) / (2 * h)
        worst[b.entry(j - b.start)] = (np.linalg.norm(fd - J[:, j]) / cn, tol)
    bad = {k: v for k, (v, tol) in worst.items() if not v <= tol}
    assert not bad, bad
