"""The product's own __host__ __device__ math (csrc/icc_camera.cuh, csrc/icc_device_math.cuh -- the functions every CUDA kernel
inlines) compiled for the CPU and checked without a GPU: camera projections against the independent NumPy models, both closed-form
Jacobians (point 2x3, intrinsics 2xK) against central finite differences for all seven models, SO(3) exp / log / Jr^-1 identities, and
the spline blending polynomials against the reference's blending matrices (SURVEY.md §8(a2) known answers) and their own derivatives,
and the trust-region controller of every LM driver (csrc/icc_trust_region.cuh) against a Python statement of Ceres' rules."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import camera_models as cm
from test_camera_models import CASES

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_math", "host_math.cu")
OUT = os.path.join(HERE, "host_math", "_build", "libhost_math.so")
DP = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def hm():
    hdrs = [os.path.join(HERE, "..", "openimucameracalibrator_b200", "csrc", f) for f in ("icc_camera.cuh", "icc_device_math.cuh", "icc_spline_chain.cuh", "icc_vision_rows.cuh", "icc_imu_rows.cuh", "icc_rotinit_math.cuh", "icc_small_linalg.cuh", "icc_points_math.cuh", "icc_trust_region.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(f) > os.path.getmtime(OUT) for f in [SRC] + hdrs):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", OUT, SRC])
    return ctypes.CDLL(OUT)


def _project(hm, model, k, p, fov=1):
    out = np.zeros(28); kk = np.zeros(10); kk[: len(k)] = k
    rc = hm.hm_project(ctypes.c_int(model), kk.ctypes.data_as(DP), np.ascontiguousarray(p, dtype=np.float64).ctypes.data_as(DP), ctypes.c_int(fov), out.ctypes.data_as(DP))
    assert rc & 2, "project() and project_with_k() disagree"
    return bool(rc & 1), out[:2].copy(), out[2:8].reshape(2, 3).copy(), out[8:].reshape(2, 10).copy()


@pytest.mark.parametrize("model,k", CASES, ids=[cm.MODEL_NAMES[m] for m, _ in CASES])
def test_device_projection_and_jacobians(hm, model, k):
    assert hm.hm_num_params(model) == cm.NUM_PARAMS[model] == len(k)
    rng = np.random.default_rng(100 + model)
    pts = np.concatenate([rng.uniform(-0.35, 0.35, (60, 2)), rng.uniform(0.3, 1.0, (60, 1))], axis=1)
    uv_ref, valid = cm.project(model, k, pts)
    for i, p in enumerate(pts):
        ok, uv, J, Jk = _project(hm, model, k, p)
        assert ok == bool(valid[i])
        if not ok:
            continue
        assert np.allclose(uv, uv_ref[i], rtol=1e-13, atol=1e-10)
        # d(u,v)/d(point): central differences on the independent NumPy model
        Jfd = np.zeros((2, 3))
        for d in range(3):
            h = 1e-6 * max(1.0, abs(p[d])); e = np.zeros(3); e[d] = h
            Jfd[:, d] = (cm.project(model, k, (p + e)[None])[0][0] - cm.project(model, k, (p - e)[None])[0][0]) / (2 * h)
        assert np.abs(J - Jfd).max() < 2e-6 * max(1.0, np.abs(Jfd).max())
        # d(u,v)/d(intrinsics)
        for q in range(len(k)):
            h = 1e-3 * abs(k[q]) if 0.0 < abs(k[q]) < 1e-4 else 1e-6 * max(1.0, abs(k[q]))   # the division distortion lives at 1e-6
            kp, km = k.copy(), k.copy(); kp[q] += h; km[q] -= h
            fd = (cm.project(model, kp, p[None])[0][0] - cm.project(model, km, p[None])[0][0]) / (2 * h)
            assert np.abs(Jk[:, q] - fd).max() < 5e-6 * max(1.0, np.abs(fd).max()), (q, Jk[:, q], fd)
        assert not Jk[:, len(k):].any()


@pytest.mark.parametrize("model,k", CASES, ids=[cm.MODEL_NAMES[m] for m, _ in CASES])
def test_device_unprojection_inverts_projection(hm, model, k):
    """unproject_gn (the un-projection of unproject_kernel / the board-pose path): project o unproject = identity for every model, and
    pixels outside a model's image are reported instead of returning garbage."""
    rng = np.random.default_rng(300 + model)
    pts = np.concatenate([rng.uniform(-0.45, 0.45, (200, 2)), np.ones((200, 1))], axis=1)
    uv, valid = cm.project(model, k, pts)
    kk = np.zeros(10); kk[: len(k)] = k
    xy = np.zeros(2)
    for i in np.flatnonzero(valid):
        ok = hm.hm_unproject(ctypes.c_int(model), kk.ctypes.data_as(DP), ctypes.c_double(uv[i, 0]), ctypes.c_double(uv[i, 1]), xy.ctypes.data_as(DP))
        assert ok and np.abs(xy - pts[i, :2]).max() < 1e-10, (i, xy, pts[i])
    if model in (cm.DOUBLE_SPHERE, cm.EXTENDED_UNIFIED):
        return                                                   # their image of the half space is unbounded in this parameter range
    ok = hm.hm_unproject(ctypes.c_int(model), kk.ctypes.data_as(DP), ctypes.c_double(1e7), ctypes.c_double(-1e7), xy.ctypes.data_as(DP))
    if ok:                                                       # if a far pixel does invert, it must invert consistently
        back, v = cm.project(model, k, np.array([[xy[0], xy[1], 1.0]]))
        assert v[0] and np.abs(back[0] - [1e7, -1e7]).max() < 1e-3


def test_fov_dispatch_switch_and_domain_checks(hm):
    ok, *_ = _project(hm, cm.FOV, np.array([437.0, 1.0, 489.0, 271.0, 0.9]), [0.1, 0.05, 0.6], fov=0)
    assert not ok                                            # the reference never dispatches FOV (residuals.h:366-389)
    ok, *_ = _project(hm, cm.DOUBLE_SPHERE, np.array([342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513]), [0.1, 0.0, -5.0])
    assert not ok
    ok, *_ = _project(hm, cm.EXTENDED_UNIFIED, np.array([438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062]), [0.1, 0.0, -5.0])
    assert not ok


def test_device_so3_functions(hm):
    rng = np.random.default_rng(7)
    for scale in (1e-12, 1e-7, 1e-3, 0.3, 2.5):
        for _ in range(20):
            w = rng.normal(0, 1, 3); w *= scale / np.linalg.norm(w)
            q = np.zeros(4); ab = np.zeros(2); back = np.zeros(3); Ji = np.zeros(9)
            hm.hm_so3_exp(w.ctypes.data_as(DP), q.ctypes.data_as(DP), ab.ctypes.data_as(DP))
            th = np.linalg.norm(w)
            assert abs(np.linalg.norm(q) - 1.0) < 1e-15 and abs(q[3] - np.cos(th / 2)) < 1e-15
            hm.hm_so3_log(q.ctypes.data_as(DP), back.ctypes.data_as(DP))
            assert np.abs(back - w).max() < 1e-14 * max(1.0, th) + 1e-22
            # Jr(w) Jr^-1(w) = I with Jr = I - a [w]x + b [w]x^2
            hm.hm_so3_jr_inv(w.ctypes.data_as(DP), Ji.ctypes.data_as(DP))
            W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            Jr = np.eye(3) - ab[0] * W + ab[1] * W @ W
            assert np.abs(Jr @ Ji.reshape(3, 3) - np.eye(3)).max() < 1e-12
            # rotation by the quaternion equals the Rodrigues matrix; qrot_inv is its transpose
            R = np.eye(3) + (np.sin(th) / th if th > 1e-9 else 1.0) * W + ((1 - np.cos(th)) / th ** 2 if th > 1e-9 else 0.5) * W @ W
            p = rng.normal(0, 1, 3); a = np.zeros(3); b = np.zeros(3)
            hm.hm_qrot(q.ctypes.data_as(DP), p.ctypes.data_as(DP), a.ctypes.data_as(DP), b.ctypes.data_as(DP))
            assert np.abs(a - R @ p).max() < 1e-14 and np.abs(b - R.T @ p).max() < 1e-14


def test_device_spline_coefficients_against_reference_blending_matrices(hm):
    # SURVEY.md §8(a2): rows = knot, columns = power of u, x120 (N = 6) / x2 (N = 3)
    M6 = np.array([[1, -5, 10, -10, 5, -1], [26, -50, 20, 20, -20, 5], [66, 0, -60, 0, 30, -10], [26, 50, 20, -20, -20, 10], [1, 5, 10, 10, 5, -5], [0, 0, 0, 0, 0, 1]]) / 120.0
    C6 = np.array([[120, 0, 0, 0, 0, 0], [119, 5, -10, 10, -5, 1], [93, 55, -30, -10, 15, -4], [27, 55, 30, -10, -15, 6], [1, 5, 10, 10, 5, -4], [0, 0, 0, 0, 0, 1]]) / 120.0
    M3 = np.array([[1, -2, 1], [1, 2, -2], [0, 0, 1]]) / 2.0

    def powers(u, n, deriv):
        out = np.zeros(n)
        for j in range(deriv, n):
            out[j] = np.prod(np.arange(j, j - deriv, -1)) * u ** (j - deriv)
        return out
    out = np.zeros(45)
    for u in (0.0, 1e-9, 0.123, 0.5, 0.987654321, 1.0, 1.02):      # u slightly above 1 occurs (row time added to normalised u, quirk q2)
        hm.hm_coeffs(ctypes.c_double(u), out.ctypes.data_as(DP))
        assert np.abs(out[0:5] - (C6 @ powers(u, 6, 0))[1:]).max() < 1e-15
        assert np.abs(out[5:10] - (C6 @ powers(u, 6, 1))[1:]).max() < 1e-14
        assert np.abs(out[10:15] - (C6 @ powers(u, 6, 2))[1:]).max() < 1e-14
        for d, sl in enumerate((slice(15, 21), slice(21, 27), slice(27, 33), slice(33, 39))):
            assert np.abs(out[sl] - M6 @ powers(u, 6, d)).max() < 1e-13
        assert np.abs(out[39:42] - M3 @ powers(u, 3, 0)).max() < 1e-15 and np.abs(out[42:45] - M3 @ powers(u, 3, 1)).max() < 1e-15
        assert abs(out[15:21].sum() - 1.0) < 1e-15 and abs(out[39:42].sum() - 1.0) < 1e-15      # partition of unity


# ---- the SO(3) spline chain of the residual kernels and its analytic knot Jacobian ----------------------------------------------------
def _qmul(a, b):
    ax, ay, az, aw = a; bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def _qexp(w):
    th = np.linalg.norm(w)
    return np.array([*(0.5 * w), 1.0]) if th < 1e-14 else np.array([*(np.sin(th / 2) / th * w), np.cos(th / 2)])


def _qlog(q):
    n = np.linalg.norm(q[:3])
    return 2.0 * q[:3] / q[3] if n < 1e-14 else 2.0 * np.arctan(n / q[3]) / n * q[:3]


def _qinv(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


_C6 = np.array([[120, 0, 0, 0, 0, 0], [119, 5, -10, 10, -5, 1], [93, 55, -30, -10, 15, -4], [27, 55, 30, -10, -15, 6], [1, 5, 10, 10, 5, -4], [0, 0, 0, 0, 0, 1]]) / 120.0


def _spline_rotation(knots, u):
    """CeresSplineHelper::evaluate_lie (basalt_spline/ceres_spline_helper.h:101-187), independent NumPy statement."""
    lam = _C6 @ np.array([u ** j for j in range(6)])
    q = knots[0].copy()
    for i in range(5):
        q = _qmul(q, _qexp(lam[i + 1] * _qlog(_qmul(_qinv(knots[i]), knots[i + 1]))))
    return q / np.linalg.norm(q)


def _chain(hm, knots, u, m):
    q = np.zeros(4); rows = np.zeros(18); du = ctypes.c_double()
    hm.hm_so3_chain(np.ascontiguousarray(knots).ctypes.data_as(DP), ctypes.c_double(u), np.ascontiguousarray(m).ctypes.data_as(DP), q.ctypes.data_as(DP), rows.ctypes.data_as(DP),
                    ctypes.byref(du))
    return q, rows.reshape(6, 3), du.value


@pytest.mark.parametrize("spread", [0.02, 0.3, 1.2], ids=["slow", "typical", "fast_rotation"])
def test_device_so3_spline_chain_and_knot_jacobian(hm, spread):
    """build_chain + so3_knot_row (the analytic Jacobian at the heart of vision_kernel / imu_kernel) against central finite differences
    of an independent NumPy statement of the cumulative SO(3) B-spline: d theta / d eps_j for right increments on every knot, and
    d theta / d u, contracted with a random row covector -- exactly what one Jacobian row of a residual needs."""
    rng = np.random.default_rng(int(spread * 100))
    for trial in range(6):
        q0 = _qexp(rng.normal(0, 1.0, 3))
        knots = [q0]
        for i in range(5):
            knots.append(_qmul(knots[-1], _qexp(rng.normal(0, spread, 3))))
        knots = np.array(knots)
        u = [0.0, 0.31, 0.77, 1.0, 1.03, 0.5][trial]                 # u > 1 occurs: the row time is added to the normalised time (quirk q2)
        m = rng.normal(0, 1, 3)
        q, rows, du = _chain(hm, knots, u, m)
        R = _spline_rotation(knots, u)
        assert min(np.abs(q - R).max(), np.abs(q + R).max()) < 1e-14
        h = 1e-6
        for j in range(6):
            for a in range(3):
                e = np.zeros(3); e[a] = h
                kp, km = knots.copy(), knots.copy()
                kp[j] = _qmul(knots[j], _qexp(e)); km[j] = _qmul(knots[j], _qexp(-e))
                dth = (_qlog(_qmul(_qinv(R), _spline_rotation(kp, u))) - _qlog(_qmul(_qinv(R), _spline_rotation(km, u)))) / (2 * h)
                assert abs(rows[j, a] - m @ dth) < 2e-8 * max(1.0, np.abs(rows).max()), (j, a, rows[j, a], m @ dth)
        dth_u = (_qlog(_qmul(_qinv(R), _spline_rotation(knots, u + h))) - _qlog(_qmul(_qinv(R), _spline_rotation(knots, u - h)))) / (2 * h)
        assert abs(du - m @ dth_u) < 2e-8 * max(1.0, abs(du))
    # a vanishing increment between two knots (identical orientations) must not produce NaNs
    knots[3] = knots[2]
    q, rows, du = _chain(hm, knots, 0.4, np.array([0.3, -0.2, 0.9]))
    assert np.isfinite(q).all() and np.isfinite(rows).all() and np.isfinite(du)


# ---- the joint x/y rows of the persistent vision kernel ------------------------------------------------------------------------------------------
_B6 = np.array([[1, -5, 10, -10, 5, -1], [26, -50, 20, 20, -20, 5], [66, 0, -60, 0, 30, -10], [26, 50, 20, -20, -20, 10], [1, 5, 10, 10, 5, -5], [0, 0, 0, 0, 0, 1]]) / 120.0


def _qmat(q):
    x, y, z, w = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _rs_pixel(model, k, so3, r3, u_so3, u_r3, T_ic, ld, X, oy):
    """RSReprojectionCostFunctorSplit (ceres_calib_split_residuals.h:319-402), independent NumPy statement: projected pixel of one corner."""
    us, ur = u_so3 + oy * ld, u_r3 + oy * ld
    R = _qmat(_spline_rotation(so3, us))
    t = (_B6 @ np.array([ur ** j for j in range(6)])) @ r3
    pi = R.T @ (X - t)
    pc = _qmat(T_ic[:4]).T @ (pi - T_ic[4:])
    uv, valid = cm.project(model, k, pc[None])
    return uv[0], bool(valid[0])


@pytest.mark.parametrize("model,k", CASES, ids=[cm.MODEL_NAMES[m] for m, _ in CASES])
def test_device_vision_rows_against_finite_differences(hm, model, k):
    """vision_corner_rows + vision_yrow_expand (icc_vision_rows.cuh: both Jacobian rows of a corner in one pass, Rodrigues-form increment
    rotations, polynomial sincos, factored y row) against central differences of the NumPy functor: right increments on the six SO(3)
    knots, the six R^3 knots, T_i_c = (upsilon, omega) of LieLocalParameterization<SE3> (ceres_local_param.h:84-115), the line delay."""
    rng = np.random.default_rng(300 + model)
    kk = np.zeros(10); kk[: len(k)] = k
    for trial in range(4):
        so3 = [_qexp(rng.normal(0, 0.6, 3))]
        for i in range(5):
            so3.append(_qmul(so3[-1], _qexp(rng.normal(0, [0.03, 0.3, 0.0, 0.8][trial], 3))))
        so3 = np.array(so3)
        r3 = rng.normal(0, 0.05, (6, 3))
        T_ic = np.concatenate([_qexp(rng.normal(0, 0.3, 3)), rng.normal(0, 0.02, 3)])
        u_so3, u_r3, ld = rng.uniform(0, 0.97), rng.uniform(0, 0.97), 6.0e-5
        # a board point about half a metre in front of the camera
        R0 = _qmat(_spline_rotation(so3, u_so3)); Ric = _qmat(T_ic[:4])
        pc = np.array([rng.uniform(-0.12, 0.12), rng.uniform(-0.08, 0.08), 0.5])
        X = R0 @ (Ric @ pc + T_ic[4:]) + (_B6 @ np.array([u_r3 ** j for j in range(6)])) @ r3
        oy = 270.0 + rng.uniform(-200, 200); ox = 480.0 + rng.uniform(-300, 300)
        rows = np.zeros(88)
        ok = hm.hm_vision_rows(ctypes.c_int(model), kk.ctypes.data_as(DP), ctypes.c_int(1), np.ascontiguousarray(so3).ctypes.data_as(DP), np.ascontiguousarray(r3).ctypes.data_as(DP),
                               ctypes.c_double(u_so3), ctypes.c_double(u_r3), T_ic.ctypes.data_as(DP), ctypes.c_double(ld), X.ctypes.data_as(DP), ctypes.c_double(ox), ctypes.c_double(oy), rows.ctypes.data_as(DP))
        uv, valid = _rs_pixel(model, k, so3, r3, u_so3, u_r3, T_ic, ld, X, oy)
        assert bool(ok) == valid
        if not valid:
            continue
        rows = rows.reshape(2, 44)
        assert np.allclose(rows[:, 43], uv - np.array([ox, oy]), rtol=1e-12, atol=1e-9)
        f = lambda s=so3, r=r3, T=T_ic, l=ld: _rs_pixel(model, k, s, r, u_so3, u_r3, T, l, X, oy)[0]   # noqa: E731
        scale = max(1.0, np.abs(rows[:, :43]).max())
        h = 1e-6
        for j in range(6):
            for a in range(3):
                e = np.zeros(3); e[a] = h
                sp, sm = so3.copy(), so3.copy(); sp[j] = _qmul(so3[j], _qexp(e)); sm[j] = _qmul(so3[j], _qexp(-e))
                assert np.abs(rows[:, 3 * j + a] - (f(s=sp) - f(s=sm)) / (2 * h)).max() < 3e-7 * scale, ("so3", j, a)
                rp, rm = r3.copy(), r3.copy(); rp[j, a] += h; rm[j, a] -= h
                assert np.abs(rows[:, 18 + 3 * j + a] - (f(r=rp) - f(r=rm)) / (2 * h)).max() < 3e-7 * scale, ("r3", j, a)
        for a in range(3):
            e = np.zeros(3); e[a] = h
            Tp, Tm = T_ic.copy(), T_ic.copy(); Tp[4:] += Ric @ e; Tm[4:] -= Ric @ e                 # translation part of T exp(delta) at delta = 0
            assert np.abs(rows[:, 36 + a] - (f(T=Tp) - f(T=Tm)) / (2 * h)).max() < 3e-7 * scale, ("upsilon", a)
            Tp, Tm = T_ic.copy(), T_ic.copy(); Tp[:4] = _qmul(T_ic[:4], _qexp(e)); Tm[:4] = _qmul(T_ic[:4], _qexp(-e))
            assert np.abs(rows[:, 39 + a] - (f(T=Tp) - f(T=Tm)) / (2 * h)).max() < 3e-7 * scale, ("omega", a)
        hl = 1e-9
        assert np.abs(rows[:, 42] - (f(l=ld + hl) - f(l=ld - hl)) / (2 * hl)).max() < 1e-5 * max(1.0, np.abs(rows[:, 42]).max()), "line delay"


def _imu_residuals(so3, r3, ba, bg, u_so3, u_r3, u_ba, u_bg, Ma, Mg, grav, w_acc, w_gyr, inv_so3_dt, inv_r3_dt, a_meas, g_meas):
    """AccelerationCostFunctorSplit / GyroCostFunctorSplit (ceres_calib_split_residuals.h:52-93,133-169), independent NumPy statement."""
    R = _qmat(_spline_rotation(so3, u_so3))
    ddc = _B6 @ np.array([0.0, 0.0, 2.0, 6.0 * u_r3, 12.0 * u_r3 ** 2, 20.0 * u_r3 ** 3])
    acc_w = inv_r3_dt ** 2 * (ddc @ r3)
    c3 = lambda u: np.array([0.5 * (1 - 2 * u + u * u), 0.5 * (1 + 2 * u - 2 * u * u), 0.5 * u * u])   # noqa: E731
    ra = w_acc * (R.T @ (acc_w + grav) - Ma @ (a_meas - c3(u_ba) @ ba))
    h = 1e-5       # body velocity = vee(R^T dR/du) / dt by central differences of the spline rotation
    om = _qlog(_qmul(_qinv(_spline_rotation(so3, u_so3 - h)), _spline_rotation(so3, u_so3 + h))) / (2 * h) * inv_so3_dt
    rg = w_gyr * (om - Mg @ (g_meas - c3(u_bg) @ bg))
    return ra, rg


def test_device_imu_rows_against_finite_differences(hm):
    """imu_accel_rows / imu_gyro_rows + the parked-row expansion (icc_imu_rows.cuh) against central differences of the NumPy functors:
    right increments on the six SO(3) knots, the six R^3 knots, gravity."""
    rng = np.random.default_rng(77)
    for trial in range(3):
        so3 = [_qexp(rng.normal(0, 0.6, 3))]
        for i in range(5):
            so3.append(_qmul(so3[-1], _qexp(rng.normal(0, [0.03, 0.3, 0.8][trial], 3))))
        so3 = np.array(so3); r3 = rng.normal(0, 0.05, (6, 3)); ba = rng.normal(0, 0.05, (3, 3)); bg = rng.normal(0, 0.01, (3, 3))
        u_so3, u_r3, u_ba, u_bg = rng.uniform(0.02, 0.97, 4)
        Ma = np.array([[1.01, -0.002, 0.003], [0, 0.99, -0.001], [0, 0, 1.02]]); Mg = np.eye(3) + rng.normal(0, 0.003, (3, 3))
        grav = np.array([0.1, -0.2, 9.8]); w_acc, w_gyr, idt_s, idt_r = 3.0, 40.0, 20.0, 20.0
        a_meas, g_meas = rng.normal(0, 3, 3), rng.normal(0, 1, 3)
        A, G = np.zeros(120), np.zeros(72)
        args = [np.ascontiguousarray(x, dtype=np.float64) for x in (so3, r3, ba, bg)]
        hm.hm_imu_rows(*[a.ctypes.data_as(DP) for a in args], *[ctypes.c_double(x) for x in (u_so3, u_r3, u_ba, u_bg)], np.ascontiguousarray(Ma).ctypes.data_as(DP), np.ascontiguousarray(Mg).ctypes.data_as(DP),
                       grav.ctypes.data_as(DP), ctypes.c_double(w_acc), ctypes.c_double(w_gyr), ctypes.c_double(idt_s), ctypes.c_double(idt_r), a_meas.ctypes.data_as(DP), g_meas.ctypes.data_as(DP),
                       A.ctypes.data_as(DP), G.ctypes.data_as(DP))
        A, G = A.reshape(3, 40), G.reshape(3, 24)
        f = lambda s=so3, r=r3, g=grav: _imu_residuals(s, r, ba, bg, u_so3, u_r3, u_ba, u_bg, Ma, Mg, g, w_acc, w_gyr, idt_s, idt_r, a_meas, g_meas)   # noqa: E731
        ra, rg = f()
        assert np.allclose(A[:, 39], ra, rtol=1e-12, atol=1e-10) and np.allclose(G[:, 18], rg, rtol=1e-7, atol=1e-7) and np.all(G[:, 19:] == 0.0)
        sa, sg = max(1.0, np.abs(A[:, :39]).max()), max(1.0, np.abs(G[:, :18]).max())
        h = 1e-6
        for j in range(6):
            for a in range(3):
                e = np.zeros(3); e[a] = h
                sp, sm = so3.copy(), so3.copy(); sp[j] = _qmul(so3[j], _qexp(e)); sm[j] = _qmul(so3[j], _qexp(-e))
                (ap, gp), (am, gm) = f(s=sp), f(s=sm)
                assert np.abs(A[:, 3 * j + a] - (ap - am) / (2 * h)).max() < 3e-7 * sa, ("acc so3", j, a)
                assert np.abs(G[:, 3 * j + a] - (gp - gm) / (2 * h)).max() < 2e-4 * sg, ("gyr so3", j, a)      # differences of a difference quotient
                rp, rm = r3.copy(), r3.copy(); rp[j, a] += h; rm[j, a] -= h
                assert np.abs(A[:, 18 + 3 * j + a] - (f(r=rp)[0] - f(r=rm)[0]) / (2 * h)).max() < 3e-7 * sa, ("acc r3", j, a)
        for a in range(3):
            e = np.zeros(3); e[a] = h
            assert np.abs(A[:, 36 + a] - (f(g=grav + e)[0] - f(g=grav - e)[0]) / (2 * h)).max() < 3e-7 * sa, ("gravity", a)


def test_device_polynomial_sincos(hm):
    s, c = ctypes.c_double(), ctypes.c_double()
    for x in np.concatenate([np.linspace(-0.7853981633974483, 0.7853981633974483, 2001), [1e-300, -1e-9, 0.9, -2.5, 40.0]]):
        hm.hm_sincos_small(ctypes.c_double(x), ctypes.byref(s), ctypes.byref(c))
        assert abs(s.value - np.sin(x)) <= 2.3e-16 * max(abs(np.sin(x)), 1e-300) + 1e-323 and abs(c.value - np.cos(x)) <= 2.3e-16


# ---- scalar pieces of the rotation / time-offset initialiser -----------------------------------------------------------------------------
def test_device_nearest_sample_rule_matches_the_reference_scan(hm):
    """FindClosestTimestamp (src/utils/utils.cc:194-212) is a linear scan keeping the FIRST strict minimum of |t - ts[i]|; the kernels use
    a bisection on the sorted times that must pick the same index, ties included."""
    rng = np.random.default_rng(11)
    ts = np.sort(rng.uniform(0, 10, 200)); ts[50] = ts[49] + 0.02; ts[51] = ts[49] + 0.04          # an exact tie candidate at the midpoint
    queries = np.concatenate([rng.uniform(-1, 11, 500), ts[:20], [ts[49] + 0.01, ts[50] + 0.01, -5.0, 50.0]])
    dist = ctypes.c_double()
    for q in queries:
        idx = hm.hm_nearest_sorted(ts.ctypes.data_as(DP), ctypes.c_int(ts.size), ctypes.c_double(q), ctypes.byref(dist))
        best, bd = 0, abs(q - ts[0])
        for i in range(1, ts.size):
            if abs(q - ts[i]) < bd:
                best, bd = i, abs(q - ts[i])
        assert idx == best and dist.value == bd


def test_device_slerp_is_eigens(hm):
    """Eigen::Quaternion::slerp (used by InterpolateQuaternions, utils.cc:234): shortest arc, linear blend when nearly parallel."""
    rng = np.random.default_rng(12)
    out = np.zeros(4)
    for trial in range(200):
        a = rng.normal(0, 1, 4); a /= np.linalg.norm(a)
        b = a + (1e-9 if trial % 5 == 0 else 1.0) * rng.normal(0, 1, 4); b /= np.linalg.norm(b)
        if trial % 3 == 0:
            b = -b                                                 # antipodal representation: slerp must take the short way
        tt = rng.uniform(0, 1)
        hm.hm_slerp4(a.ctypes.data_as(DP), b.ctypes.data_as(DP), ctypes.c_double(tt), out.ctypes.data_as(DP))
        d = float(a @ b); ad = abs(d)
        if ad >= 1.0 - np.finfo(float).eps:
            s0, s1 = 1.0 - tt, tt
        else:
            th = np.arccos(ad); s0, s1 = np.sin((1 - tt) * th) / np.sin(th), np.sin(tt * th) / np.sin(th)
        ref = s0 * a + (-s1 if d < 0 else s1) * b
        assert np.abs(out - ref).max() < 1e-15
        if ad < 1.0 - 1e-6:
            assert abs(np.linalg.norm(out) - 1.0) < 1e-12          # stays on the unit sphere on a proper arc


def test_device_dominant_eigenvector_of_horns_matrix(hm):
    """eig4_max (cyclic Jacobi) behind the closed-form rotation of the golden-section objective: the eigenvector of the largest eigenvalue
    of a symmetric 4x4 matrix, against numpy.linalg.eigh; and the rotation it encodes maximises tr(R M) like the reference's SVD route."""
    rng = np.random.default_rng(13)
    q = np.zeros(4)
    for trial in range(100):
        M = rng.normal(0, 1, (3, 3))                                # sum of imu x vis outer products
        Sxx, Sxy, Sxz, Syx, Syy, Syz, Szx, Szy, Szz = M.ravel()
        N = np.array([[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx], [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
                      [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy], [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]])
        hm.hm_eig4_max(np.ascontiguousarray(N).ctypes.data_as(DP), q.ctypes.data_as(DP))
        w, V = np.linalg.eigh(N)
        v = V[:, -1]
        assert abs(np.linalg.norm(q) - 1.0) < 1e-12 and min(np.abs(q - v).max(), np.abs(q + v).max()) < 1e-9 / max(w[-1] - w[-2], 1e-3)
        assert abs(q @ N @ q - w[-1]) < 1e-10 * max(1.0, abs(w[-1]))


# ---- small dense linear algebra of the upstream kernels -------------------------------------------------------------------------------
CHOL_SIZES = [3, 6, 8, 10, 12]


@pytest.mark.parametrize("n", CHOL_SIZES)
def test_device_cholesky_solve(hm, n):
    """chol_solve<N> (3x3 point systems, 6x6 pose systems, 8x8 homography normal equations, 10x10 reduced intrinsics
    systems, 12x12 static IMU steps) against numpy.linalg.solve; an indefinite matrix is reported instead of producing NaNs."""
    rng = np.random.default_rng(20 + n)
    for trial in range(50):
        G = rng.normal(0, 1, (n + 3, n)); A = G.T @ G * 10.0 ** rng.uniform(-3, 3)
        b = rng.normal(0, 1, n); x = b.copy()
        assert hm.hm_chol_solve(ctypes.c_int(n), np.ascontiguousarray(A).ctypes.data_as(DP), x.ctypes.data_as(DP)) == 1
        ref = np.linalg.solve(A, b)
        assert np.abs(x - ref).max() < 1e-9 * np.linalg.cond(A) * max(1e-12, np.abs(ref).max()) + 1e-300
    A = np.eye(n); A[n - 1, n - 1] = -1.0
    x = np.ones(n)
    assert hm.hm_chol_solve(ctypes.c_int(n), A.ctypes.data_as(DP), x.ctypes.data_as(DP)) == 0 and np.isfinite(x).all()


@pytest.mark.parametrize("n", CHOL_SIZES)
def test_device_cholesky_factor_once_substitute_many(hm, n):
    """chol_factor<N> once, chol_substitute<N> per right-hand side (the camera calibration's 11 columns per view): every column
    against numpy.linalg.solve and equal, bit for bit, to chol_solve<N> of that column alone; an indefinite matrix is reported with
    finite output in every column."""
    rng = np.random.default_rng(40 + n)
    nrhs = 11
    for trial in range(20):
        G = rng.normal(0, 1, (n + 3, n)); A = np.ascontiguousarray(G.T @ G * 10.0 ** rng.uniform(-3, 3))
        B = rng.normal(0, 1, (nrhs, n)); X = B.copy()
        assert hm.hm_chol_factor_substitute(ctypes.c_int(n), A.ctypes.data_as(DP), ctypes.c_int(nrhs), X.ctypes.data_as(DP)) == 1
        ref = np.linalg.solve(A, B.T).T
        assert np.abs(X - ref).max() < 1e-9 * np.linalg.cond(A) * max(1e-12, np.abs(ref).max()) + 1e-300
        for r in range(nrhs):
            x = B[r].copy()
            assert hm.hm_chol_solve(ctypes.c_int(n), A.ctypes.data_as(DP), x.ctypes.data_as(DP)) == 1
            assert np.array_equal(x, X[r])
    A = np.eye(n); A[n // 2, n // 2] = -1.0
    X = np.ones((nrhs, n))
    assert hm.hm_chol_factor_substitute(ctypes.c_int(n), A.ctypes.data_as(DP), ctypes.c_int(nrhs), X.ctypes.data_as(DP)) == 0 and np.isfinite(X).all()


def test_device_quaternion_from_rotation_matrix(hm):
    """quat_from_columns (pose from the homography): all four branches of the trace / largest-diagonal rule give q with R(q) = R."""
    rng = np.random.default_rng(31)
    q = np.zeros(4)
    axes = [rng.normal(0, 1, 3) for _ in range(60)] + [np.array([np.pi, 0, 0]), np.array([0, np.pi, 0]), np.array([0, 0, np.pi]), np.array([1e-9, 0, 0])]
    for w in axes:
        th = np.linalg.norm(w); W = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        R = np.eye(3) + (np.sin(th) / th) * W + ((1 - np.cos(th)) / th ** 2) * W @ W
        hm.hm_quat_from_columns(np.ascontiguousarray(R).ctypes.data_as(DP), q.ctypes.data_as(DP))
        x, y, z, s = q
        Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * s), 2 * (x * z + y * s)], [2 * (x * y + z * s), 1 - 2 * (x * x + z * z), 2 * (y * z - x * s)],
                       [2 * (x * z - y * s), 2 * (y * z + x * s), 1 - 2 * (x * x + y * y)]])
        assert abs(np.linalg.norm(q) - 1.0) < 1e-14 and np.abs(Rq - R).max() < 1e-12


def test_device_homogeneous_point_parameterization(hm):
    """ceres::HomogeneousVectorParameterization(4) as icc_points.cu uses it (icc_points_math.cuh): Plus against the NumPy statement of
    tests/helpers.py (all branches of the Householder vector: w > 0, w <= 0, x on the w axis), Plus keeps |x|, Plus(x, 0) = x, the local
    Jacobian against central differences of Plus, and the de-homogenised point."""
    from helpers import plus_homog4
    rng = np.random.default_rng(41)
    xs = [rng.normal(0, 1, 4) * 10.0 ** rng.uniform(-2, 2) for _ in range(40)]
    xs += [np.array([0.3, -0.2, 0.1, 1.0]), np.array([0.3, -0.2, 0.1, -1.0]), np.array([0.0, 0.0, 0.0, 2.0]), np.array([0.0, 0.0, 0.0, -2.0]), np.array([1e-9, 0.0, 0.0, 1.0])]
    out, board, jac = np.zeros(4), np.zeros(4), np.zeros(12)
    for x in xs:
        x = np.ascontiguousarray(x)
        for d in (rng.normal(0, 0.3, 3), rng.normal(0, 1e-6, 3), np.zeros(3), np.array([3.0, -2.0, 1.0])):
            d = np.ascontiguousarray(d)
            hm.hm_points_plus(x.ctypes.data_as(DP), d.ctypes.data_as(DP), out.ctypes.data_as(DP))
            ref = plus_homog4(x, d)
            assert np.abs(out - ref).max() <= 1e-14 * np.linalg.norm(x), (x, d, out, ref)
            assert abs(np.linalg.norm(out) - np.linalg.norm(x)) <= 1e-14 * np.linalg.norm(x)
        hm.hm_points_prepare(x.ctypes.data_as(DP), board.ctypes.data_as(DP), jac.ctypes.data_as(DP))
        assert np.allclose(board, [x[0] / x[3], x[1] / x[3], x[2] / x[3], 1.0], rtol=1e-15, atol=0)
        J = jac.reshape(4, 3); eps = 1e-6
        for i in range(3):
            e = np.zeros(3); e[i] = eps
            fd = (plus_homog4(x, e) - plus_homog4(x, -e)) / (2 * eps)
            assert np.abs(J[:, i] - fd).max() <= 1e-8 * np.linalg.norm(x), (x, i, J[:, i], fd)
        if x[:3] @ x[:3] > np.finfo(float).eps:                                # (Ceres' own shortcut for x on the w axis takes H = I there)
            assert np.abs(J.T @ x).max() <= 1e-14 * (x @ x)                   # the tangent columns are orthogonal to x


# ---- the trust-region controller shared by every LM driver (icc_trust_region.cuh) ---------------------------------------------------------
class _TrRules:
    """Ceres 2.1 TrustRegionMinimizer step control, independent statement: the state the controller must hold after every call."""

    def __init__(self, ftol, ptol, gtol, r0, rmax, rmin, eta, max_it, max_invalid, check):
        self.o = dict(ftol=ftol, ptol=ptol, gtol=gtol, rmax=rmax, rmin=rmin, eta=eta, max_it=max_it, max_invalid=max_invalid, check=check)
        self.radius, self.nu, self.cost, self.initial_cost, self.mc = r0, 2.0, 0.0, 0.0, 0.0
        self.invalid = self.iterations = self.successful = 0
        self.term, self.stale = -1, 1

    def state(self):
        return [self.radius, self.nu, self.cost, self.initial_cost, self.invalid, self.iterations, self.successful, self.term, self.stale]

    def _shrink(self):
        self.radius /= self.nu; self.nu *= 2.0
        if self.radius < self.o["rmin"]:
            self.term = 4

    def cont(self):
        if self.term < 0 and self.iterations >= self.o["max_it"]:
            self.term = 0
        return self.term < 0

    def jacobian(self, cost, gmax):
        self.cost = cost; self.stale = 0
        if self.iterations == 0:
            self.initial_cost = cost
        if self.o["check"] and gmax <= self.o["gtol"]:
            self.term = 3
        return self.term < 0

    def step(self, valid, mc, sn, xn):
        self.iterations += 1
        if not valid or not mc > 0.0:
            self.invalid += 1
            if self.invalid >= self.o["max_invalid"]:
                self.term = 4
            else:
                self._shrink()
            return False
        self.invalid, self.mc = 0, mc
        if self.o["check"] and sn <= self.o["ptol"] * (xn + self.o["ptol"]):
            self.term = 2
            return False
        return True

    def candidate(self, c):
        c = c if np.isfinite(c) else np.finfo(float).max
        change = self.cost - c
        if self.o["check"] and abs(change) <= self.o["ftol"] * self.cost:
            self.term = 1
            return False
        rho = change / self.mc
        if not rho > self.o["eta"]:
            self._shrink()
            return False
        self.successful += 1; self.cost = c; self.nu = 2.0; self.stale = 1
        self.radius = min(self.o["rmax"], self.radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
        return True


class _Tr:
    """The product's controller and _TrRules driven in lockstep; every call must return the same and leave the same state."""

    def __init__(self, hm, ftol=1e-6, ptol=1e-8, gtol=1e-10, r0=1e4, rmax=1e16, rmin=1e-32, eta=1e-3, max_it=50, max_invalid=5, check=1):
        self.hm, self.buf = hm, ctypes.create_string_buffer(hm.hm_tr_size())
        d = np.array([ftol, ptol, gtol, r0, rmax, rmin, eta]); i = np.array([max_it, max_invalid, check], dtype=np.int32)
        hm.hm_tr_start(self.buf, d.ctypes.data_as(DP), i.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
        self.ref = _TrRules(ftol, ptol, gtol, r0, rmax, rmin, eta, max_it, max_invalid, check)
        self._check(True, True)

    def state(self):
        s = np.zeros(9); self.hm.hm_tr_state(self.buf, s.ctypes.data_as(DP))
        return s

    def _check(self, got, want):
        assert bool(got) == want and list(self.state()) == self.ref.state(), (bool(got), want, list(self.state()), self.ref.state())
        return want

    def cont(self):
        return self._check(self.hm.hm_tr_continue(self.buf), self.ref.cont())

    def jacobian(self, cost, gmax):
        return self._check(self.hm.hm_tr_jacobian(self.buf, ctypes.c_double(cost), ctypes.c_double(gmax)), self.ref.jacobian(cost, gmax))

    def step(self, valid, mc, sn=1.0, xn=1.0):
        return self._check(self.hm.hm_tr_step(self.buf, ctypes.c_int(int(valid)), ctypes.c_double(mc), ctypes.c_double(sn), ctypes.c_double(xn)), self.ref.step(valid, mc, sn, xn))

    def candidate(self, c):
        return self._check(self.hm.hm_tr_candidate(self.buf, ctypes.c_double(c)), self.ref.candidate(c))

    def get(self, name):
        return self.state()[["radius", "nu", "cost", "initial_cost", "invalid", "iterations", "successful", "termination", "stale"].index(name)]


def test_trust_region_invalid_steps_shrink_and_stop_at_max_invalid(hm):
    t = _Tr(hm)
    assert t.cont() and t.jacobian(10.0, 1.0)
    for k in range(4):
        assert not t.step(False, 1.0) and t.cont()
        assert t.get("radius") == 1e4 / 2.0 ** ((k + 1) * (k + 2) // 2) and t.get("nu") == 2.0 ** (k + 2)   # r / 2, / 4, / 8, ...
    assert not t.step(True, -1.0) and not t.cont()            # no model decrease: the fifth invalid step in a row
    assert t.get("termination") == 4 and t.get("iterations") == 5 and t.get("successful") == 0 and t.get("radius") == 1e4 / 1024.0


def test_trust_region_min_radius_after_invalid_and_after_rejected_steps(hm):
    t = _Tr(hm, r0=1.0, rmin=0.3)
    assert t.cont() and t.jacobian(10.0, 1.0)
    assert not t.step(False, 1.0) and t.get("radius") == 0.5 and t.cont()
    assert not t.step(False, 1.0) and t.get("radius") == 0.125 and not t.cont() and t.get("termination") == 4 and t.get("invalid") == 2
    t = _Tr(hm, r0=1.0, rmin=0.3)
    assert t.cont() and t.jacobian(10.0, 1.0)
    assert t.step(True, 1.0) and not t.candidate(10.5) and t.get("radius") == 0.5 and t.cont()   # cost went up: rejected
    assert t.step(True, 1.0) and not t.candidate(np.nan) and t.get("radius") == 0.125 and not t.cont() and t.get("termination") == 4
    assert t.get("successful") == 0 and t.get("cost") == 10.0


def test_trust_region_accepted_steps_grow_the_radius_up_to_max_radius(hm):
    t = _Tr(hm, r0=1.0, rmax=5.0)
    assert t.cont() and t.jacobian(10.0, 1.0)
    assert t.step(True, 2.0) and t.candidate(8.0)              # rho = 1: radius x 3
    assert t.get("radius") == 3.0 and t.get("stale") == 1 and t.get("cost") == 8.0 and t.get("successful") == 1
    assert t.cont() and t.jacobian(8.0, 1.0) and t.step(True, 2.0) and t.candidate(6.0)
    assert t.get("radius") == 5.0 and t.get("nu") == 2.0       # 9 capped at max_radius
    assert t.cont() and t.jacobian(6.0, 1.0) and t.step(True, 2.0) and t.candidate(5.5)   # rho = 0.25: radius / max(1/3, 1.125)
    assert t.get("radius") == 5.0 / 1.125 and t.get("initial_cost") == 10.0


def test_trust_region_gradient_stop_on_the_first_jacobian(hm):
    t = _Tr(hm)
    assert t.cont() and not t.jacobian(3.0, 1e-11) and not t.cont()
    assert t.get("termination") == 3 and t.get("iterations") == 0 and t.get("initial_cost") == 3.0 and t.get("cost") == 3.0


def test_trust_region_function_and_parameter_tolerance_stops_accept_nothing(hm):
    t = _Tr(hm, ftol=1e-6)
    assert t.cont() and t.jacobian(1.0, 1.0) and t.step(True, 1e-3)
    assert not t.candidate(1.0 - 5e-7) and not t.cont()
    assert t.get("termination") == 1 and t.get("successful") == 0 and t.get("cost") == 1.0 and t.get("iterations") == 1
    t = _Tr(hm, ptol=1e-8)
    assert t.cont() and t.jacobian(1.0, 1.0) and t.step(True, 0.5) and t.candidate(0.5)
    assert t.cont() and t.jacobian(0.5, 1.0) and not t.step(True, 0.1, sn=1e-8 * 2.0, xn=2.0) and not t.cont()
    assert t.get("termination") == 2 and t.get("successful") == 1 and t.get("cost") == 0.5 and t.get("iterations") == 2


def test_trust_region_without_convergence_tests(hm):
    """icc_lm_iterations' fixed-count runs: no gradient, parameter or function stop; the iteration limit, invalid steps and the
    minimum radius still stop the run."""
    t = _Tr(hm, max_it=4, check=0)
    assert t.cont() and t.jacobian(1.0, 0.0)
    assert t.step(True, 1.0, sn=0.0) and not t.candidate(1.0) and t.cont()   # zero step, unchanged cost: rejected
    assert t.step(True, 1.0, sn=0.0) and t.candidate(0.0) and t.cont()
    assert t.jacobian(0.0, 0.0) and t.step(True, 1.0) and not t.candidate(0.0) and t.cont()
    assert not t.step(False, 1.0) and not t.cont() and t.get("termination") == 0 and t.get("iterations") == 4
    t = _Tr(hm, check=0, max_invalid=2)
    assert t.cont() and t.jacobian(1.0, 0.0) and not t.step(False, 0.0) and t.cont() and not t.step(True, np.nan) and not t.cont()
    assert t.get("termination") == 4
    t = _Tr(hm, check=0, r0=1.0, rmin=0.4)
    assert t.cont() and t.jacobian(1.0, 0.0) and t.step(True, 1.0) and not t.candidate(2.0) and t.cont()
    assert t.step(True, 1.0) and not t.candidate(2.0) and not t.cont() and t.get("termination") == 4


@pytest.mark.filterwarnings("ignore::RuntimeWarning")             # the rules overflow to inf on huge candidate costs, as the C++ does
def test_trust_region_random_sequences_follow_the_rules(hm):
    """Random mixes of invalid, rejected, accepted and converged steps, the controller against the rules after every call."""
    rng = np.random.default_rng(5)
    for trial in range(300):
        t = _Tr(hm, ftol=10.0 ** rng.uniform(-8, -2), ptol=10.0 ** rng.uniform(-10, -4), r0=10.0 ** rng.uniform(-2, 4), rmax=10.0 ** rng.uniform(0, 6),
                rmin=10.0 ** rng.uniform(-8, -1), max_it=int(rng.integers(0, 30)), max_invalid=int(rng.integers(1, 6)), check=int(rng.integers(0, 2)))
        cost = rng.uniform(1.0, 10.0)
        while t.cont():
            if t.get("stale") and not t.jacobian(cost, 10.0 ** rng.uniform(-12, 0)):
                break
            mc = rng.choice([-1.0, 0.0, np.nan, rng.uniform(0.0, 0.5) * cost])
            if t.step(rng.uniform() > 0.15, mc, 10.0 ** rng.uniform(-12, 0), rng.uniform(0, 10)):
                c = rng.choice([cost * (1 + rng.normal(0, 1e-7)), cost - mc * rng.uniform(-1, 2), np.inf, np.nan])
                if t.candidate(c):
                    cost = c
        assert t.get("termination") in (0, 1, 2, 3, 4)
