"""The local tangent reprojection error of the spline solve (icc_set_reprojection_error(ICC_REPROJ_ERROR_TANGENT), `--reprojection_error
tangent`): every corner is its unit bearing b, and the predicted camera-frame point p scores r = s (e1.p, e2.p) / (b.p).

CPU part: the product's tangent rows (icc_vision_rows.cuh, compiled for the CPU by tests/tangent_spline/) against central differences of
the same residual, for DoubleSphere and ExtendedUnified corners 90-105 degrees off-axis and the line-delay column; the failure rules; the
first-order equivalence with the pixel residual of a pinhole corner near the principal point; the scale s against a NumPy derivative; the
oracle's tangent functor against a NumPy statement and its gradient against central differences; the API and CLI rules.
GPU part (-m gpu): cost, residuals, J^T r and J^T J against the oracle for every camera model through both Jacobian paths; the two-stage
LM against the oracle on a small problem and on config 4; a wide-lens sequence with corners past 90 degrees; the default is unchanged;
the CLI chain; the sharded solve."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from helpers import F_STAGE1, F_STAGE2, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_scaled_parity
from test_camera_models import CASES
from test_host_device_math import _B6, _qexp, _qmat, _qmul, _spline_rotation
from wide_angle_support import oracle_bearings

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
POSE_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "estimate_camera_poses_from_checkerboard")
DP = ctypes.POINTER(ctypes.c_double)
W, H = 960, 540
# wide lenses whose image corners are ~100 degrees off-axis (as in test_wide_angle_poses)
WIDE = [(cm.DOUBLE_SPHERE, np.array([200.0, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513])),
        (cm.EXTENDED_UNIFIED, np.array([250.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062]))]
ALL_IDS = [cm.MODEL_NAMES[m] for m, _ in CASES]
_LIB = None


def ts():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_tangent_spline_"), "libtangent_rows.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "tangent_spline", "tangent_rows_host_math.cu")])
        _LIB = ctypes.CDLL(out)
        _LIB.ts_tangent_scale.restype = ctypes.c_double
    return _LIB


def _p(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(DP)


def numpy_scale(model, k):
    """sqrt(|det d(u,v)/d(x,y)|) of the NumPy camera model at the principal ray, by Richardson-extrapolated central differences."""
    def D(h):
        J = np.zeros((2, 2))
        for a in range(2):
            e = np.zeros(3); e[a] = h
            pp, _ = cm.project(model, k, (np.array([0.0, 0.0, 1.0]) + e)[None])
            pm, _ = cm.project(model, k, (np.array([0.0, 0.0, 1.0]) - e)[None])
            J[:, a] = (pp[0] - pm[0]) / (2 * h)
        return J
    J = (4 * D(5e-5) - D(1e-4)) / 3
    return float(np.sqrt(abs(np.linalg.det(J))))


def closed_scale(model, k):
    """the same scale in closed form: J0 = m [[f, skew], [0, f aspect]] with m = 1, except FOV (2 tan(w/2) / w) and DoubleSphere (1 / (1 + xi))"""
    f, aspect = k[0], k[1]
    m = {cm.FOV: 2.0 * np.tan(0.5 * k[4]) / k[4] if len(k) > 4 else 1.0, cm.DOUBLE_SPHERE: 1.0 / (1.0 + k[5]) if len(k) > 5 else 1.0}.get(model, 1.0)
    return float(f * np.sqrt(aspect) * abs(m))


def _state(rng, spread=0.3):
    so3 = [_qexp(rng.normal(0, 0.6, 3))]
    for _ in range(5):
        so3.append(_qmul(so3[-1], _qexp(rng.normal(0, spread, 3))))
    return np.array(so3), rng.normal(0, 0.05, (6, 3)), np.concatenate([_qexp(rng.normal(0, 0.3, 3)), rng.normal(0, 0.02, 3)])


def _point_for(pc, so3, r3, T_ic, u_so3, u_r3, ld, oy):
    """board point whose camera-frame coordinates at the corner's row time are pc"""
    us, ur = u_so3 + oy * ld, u_r3 + oy * ld
    return _qmat(_spline_rotation(so3, us)) @ (_qmat(T_ic[:4]) @ pc + T_ic[4:]) + (_B6 @ np.array([ur ** j for j in range(6)])) @ r3


def _rows(so3, r3, u_so3, u_r3, T_ic, ld, X, oy, b, ok, s):
    rows = np.zeros(88)
    st = ts().ts_tangent_rows(_p(so3), _p(r3), ctypes.c_double(u_so3), ctypes.c_double(u_r3), _p(T_ic), ctypes.c_double(ld), _p(X), ctypes.c_double(oy),
                              _p(b), ctypes.c_int(int(ok)), ctypes.c_double(s), rows.ctypes.data_as(DP))
    return st, rows.reshape(2, 44)


# ---- CPU: the product's rows -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,k", WIDE, ids=["DOUBLE_SPHERE", "EXTENDED_UNIFIED"])
def test_tangent_rows_against_central_differences_past_90_degrees(model, k):
    rng = np.random.default_rng(500 + model)
    s = ts().ts_tangent_scale(model, _p(np.pad(k, (0, 10 - len(k)))), 1)
    n_checked = 0
    for trial in range(6):
        so3, r3, T_ic = _state(rng, [0.03, 0.3, 0.8][trial % 3])
        u_so3, u_r3, ld = rng.uniform(0, 0.97), rng.uniform(0, 0.97), 6.0e-5
        th, ph = np.radians(rng.uniform(90.0, 105.0)), rng.uniform(0, 2 * np.pi)
        d = np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
        pc = 0.5 * d
        px, valid = cm.project(model, k, (d + rng.normal(0, 3e-3, 3))[None])      # the observed corner: a ray near the prediction
        if not valid[0]:
            continue
        b, ok = oracle_bearings(model, k, px)
        assert ok[0] and np.degrees(np.arccos(b[0, 2])) > 85.0
        oy = float(px[0, 1])
        X = _point_for(pc, so3, r3, T_ic, u_so3, u_r3, ld, oy)
        st, rows = _rows(so3, r3, u_so3, u_r3, T_ic, ld, X, oy, b[0], 1, s)
        assert st == 1 and np.abs(rows[:, 43]).max() > 1e-3 and np.abs(rows[:, :43]).max() > 0
        f = lambda sq=so3, r=r3, T=T_ic, l=ld: _rows(sq, r, u_so3, u_r3, T, l, X, oy, b[0], 1, s)[1][:, 43]   # noqa: E731
        scale = max(1.0, np.abs(rows[:, :43]).max())
        h = 1e-6
        Ric = _qmat(T_ic[:4])
        for j in range(6):
            for a in range(3):
                e = np.zeros(3); e[a] = h
                sp, sm = so3.copy(), so3.copy(); sp[j] = _qmul(so3[j], _qexp(e)); sm[j] = _qmul(so3[j], _qexp(-e))
                assert np.abs(rows[:, 3 * j + a] - (f(sq=sp) - f(sq=sm)) / (2 * h)).max() < 3e-7 * scale, ("so3", j, a)
                rp, rm = r3.copy(), r3.copy(); rp[j, a] += h; rm[j, a] -= h
                assert np.abs(rows[:, 18 + 3 * j + a] - (f(r=rp) - f(r=rm)) / (2 * h)).max() < 3e-7 * scale, ("r3", j, a)
        for a in range(3):
            e = np.zeros(3); e[a] = h
            Tp, Tm = T_ic.copy(), T_ic.copy(); Tp[4:] += Ric @ e; Tm[4:] -= Ric @ e
            assert np.abs(rows[:, 36 + a] - (f(T=Tp) - f(T=Tm)) / (2 * h)).max() < 3e-7 * scale, ("upsilon", a)
            Tp, Tm = T_ic.copy(), T_ic.copy(); Tp[:4] = _qmul(T_ic[:4], _qexp(e)); Tm[:4] = _qmul(T_ic[:4], _qexp(-e))
            assert np.abs(rows[:, 39 + a] - (f(T=Tp) - f(T=Tm)) / (2 * h)).max() < 3e-7 * scale, ("omega", a)
        hl = 1e-9
        assert np.abs(rows[:, 42] - (f(l=ld + hl) - f(l=ld - hl)) / (2 * hl)).max() < 1e-5 * max(1.0, np.abs(rows[:, 42]).max()), "line delay"
        assert np.abs(rows[:, 42]).max() > 0
        n_checked += 1
    assert n_checked >= 4


def test_tangent_rows_failure_rules():
    rng = np.random.default_rng(3)
    so3, r3, T_ic = _state(rng)
    pc = np.array([0.1, -0.05, 0.5]); oy = 200.0
    X = _point_for(pc, so3, r3, T_ic, 0.3, 0.6, 5e-5, oy)
    b = pc / np.linalg.norm(pc) + np.array([0.01, 0.0, 0.0]); b /= np.linalg.norm(b)
    st, rows = _rows(so3, r3, 0.3, 0.6, T_ic, 5e-5, X, oy, b, 0, 400.0)          # no bearing: zero residual, zero rows
    assert st == -1 and not rows.any()
    st, rows = _rows(so3, r3, 0.3, 0.6, T_ic, 5e-5, X, oy, -b, 1, 400.0)         # prediction behind the ray: q12's constant
    assert st == 0 and (rows[:, 43] == 1e10).all() and not rows[:, :43].any()
    st, rows = _rows(so3, r3, 0.3, 0.6, T_ic, 5e-5, X, oy, b, 1, 400.0)
    assert st == 1 and np.abs(rows[:, :43]).max() > 0


def test_tangent_matches_pixel_residual_to_first_order_at_the_principal_point():
    k = np.array([437.0, 1.0, 0.0, 489.0, 271.0, 0.0, 0.0])
    k10 = np.pad(k, (0, 3))
    s = ts().ts_tangent_scale(cm.PINHOLE, _p(k10), 1)
    assert abs(s - 437.0) < 1e-12 * 437.0
    rng = np.random.default_rng(11)
    so3, r3, T_ic = _state(rng)
    u1, u2 = rng.normal(size=2), rng.normal(size=2)
    diffs = []
    for rho in (2.0, 0.2, 0.02):
        obs = np.array([489.0, 271.0]) + rho * u1                # observed corner and prediction within a few pixels of the centre
        pred = np.array([489.0, 271.0]) + rho * u2
        pc = 0.5 * np.array([(pred[0] - 489.0) / 437.0, (pred[1] - 271.0) / 437.0, 1.0])
        X = _point_for(pc, so3, r3, T_ic, 0.4, 0.5, 6e-5, obs[1])
        b, ok = oracle_bearings(cm.PINHOLE, k, obs[None])
        st, rt = _rows(so3, r3, 0.4, 0.5, T_ic, 6e-5, X, obs[1], b[0], ok[0], s)
        rp = np.zeros(88)
        assert ts().ts_pixel_rows(cm.PINHOLE, _p(k10), _p(so3), _p(r3), ctypes.c_double(0.4), ctypes.c_double(0.5), _p(T_ic), ctypes.c_double(6e-5), _p(X),
                                  ctypes.c_double(obs[0]), ctypes.c_double(obs[1]), rp.ctypes.data_as(DP)) == 1
        rp = rp.reshape(2, 44)
        assert st == 1 and np.abs(rp[:, 43] - rho * (u2 - u1)).max() < 1e-9
        d = np.abs(rt[:, 43] - rp[:, 43]).max()
        assert d <= 5.0 * rho ** 2 / 437.0, (rho, d)
        diffs.append(d)
        assert np.abs(rt[:, :42] - rp[:, :42]).max() <= 5e-2 * np.abs(rp[:, :42]).max()   # the rows agree to O(|offset| / f)
    assert diffs[1] < 0.05 * diffs[0] and diffs[2] < 0.05 * diffs[1]                     # quadratic, not linear, in |r|


@pytest.mark.parametrize("model,k", CASES + WIDE, ids=ALL_IDS + ["wide_DOUBLE_SPHERE", "wide_EXTENDED_UNIFIED"])
def test_tangent_scale_against_numpy(model, k):
    s = ts().ts_tangent_scale(model, _p(np.pad(k, (0, 10 - len(k)))), 1)
    assert abs(s - closed_scale(model, k)) < 1e-13 * s
    assert abs(s - numpy_scale(model, k)) < 1e-7 * s            # (cancellation in the division model's NumPy inverse limits the difference quotient)


# ---- CPU: the oracle ---------------------------------------------------------------------------------------------------------------------
_ORACLE = None


def new_tangent_oracle():
    """the CPU oracle with its vision functor able to score bearings (tests/tangent_spline/tangent_oracle.cpp), built once per process"""
    global _ORACLE
    if _ORACLE is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_tangent_oracle_"), "libicc_tangent_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(HERE, "tangent_spline", "tangent_oracle.cpp")])
        _ORACLE = ctypes.CDLL(out)
    return capi.CApi(_ORACLE, "icco_", 0)


def tangent_oracle(ds):
    """the oracle on `ds` with the NumPy bearings and scale (independent of the product)"""
    o = new_tangent_oracle(); capi.load_dataset(o, ds)
    set_oracle_bearings(o, ds)
    return o


def pixel_mean_reproj(o, ds):
    """the oracle's mean pixel reprojection error at its current state (what the product reports in either mode)"""
    o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], 0, None, None, 0.0)
    e = o.mean_reprojection_error()
    set_oracle_bearings(o, ds)
    return e


def set_oracle_bearings(o, ds):
    b, ok = oracle_bearings(ds["model"], ds["intrinsics"], ds["uv"])
    b = np.ascontiguousarray(b, dtype=np.float64); ok = np.ascontiguousarray(ok, dtype=np.int32)
    o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], len(ok), b.ctypes.data_as(DP),
            ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), closed_scale(ds["model"], ds["intrinsics"]))
    return b, ok


def test_tangent_oracle_keeps_the_pixel_functor(oracle_factory):
    """without bearings the tangent oracle is the oracle: bit-identical evaluation and LM"""
    ds = syn.make_dataset(syn.tiny_config(*WIDE[0]))
    a, b = oracle_factory(), new_tangent_oracle()
    capi.load_dataset(a, ds); capi.load_dataset(b, ds)
    for x, y in zip(a.evaluate(F_STAGE1, hessian=True), b.evaluate(F_STAGE1, hessian=True)):
        assert np.array_equal(x, y)
    sa, sb = a.lm_iterations(3, F_STAGE1), b.lm_iterations(3, F_STAGE1)
    assert sa.final_cost == sb.final_cost and np.array_equal(a.get_T_i_c(), b.get_T_i_c())


def test_oracle_tangent_functor_against_numpy():
    """With a distortion-free pinhole, the pixel functor's prediction gives each corner's predicted ray; the NumPy tangent error of that
    ray against the NumPy bearing must equal the oracle's tangent residual."""
    k = (437.0, 1.0, 0.0, 489.0, 271.0, 0.0, 0.0)
    ds = syn.make_dataset(syn.tiny_config(cm.PINHOLE, k))
    o = new_tangent_oracle(); capi.load_dataset(o, ds)
    nv = o.num_residuals()[0]
    assert nv == ds["uv"].size                                       # every corner is used, in input order
    rp = o.evaluate(F_STAGE1, gradient=False)[1][:nv].reshape(-1, 2)
    b, ok = set_oracle_bearings(o, ds)
    rt = o.evaluate(F_STAGE1, gradient=False)[1][:nv].reshape(-1, 2)
    pred = rp + ds["uv"]
    d = np.stack([(pred[:, 0] - 489.0) / 437.0, (pred[:, 1] - 271.0) / 437.0, np.ones(len(pred))], -1)
    sg = np.where(b[:, 2] < 0, -1.0, 1.0); a = -1.0 / (sg + b[:, 2]); c = b[:, 0] * b[:, 1] * a
    e1 = np.stack([1 + sg * b[:, 0] ** 2 * a, sg * c, -sg * b[:, 0]], -1); e2 = np.stack([c, sg + b[:, 1] ** 2 * a, -b[:, 1]], -1)
    bd = np.sum(b * d, 1)
    ref = 437.0 * np.stack([np.sum(e1 * d, 1) / bd, np.sum(e2 * d, 1) / bd], -1)
    assert ok.all() and np.abs(rt - ref).max() < 1e-9 * np.abs(ref).max()
    assert pixel_mean_reproj(o, ds) == pytest.approx(np.mean(np.linalg.norm(rp, axis=1)), rel=1e-12)


def test_oracle_tangent_gradient_against_central_differences():
    model, k = WIDE[0]
    ds = syn.make_dataset(syn.tiny_config(model, k))
    o = tangent_oracle(ds)
    flags = capi.FLAG_T_I_C | capi.FLAG_CAM_LINE_DELAY
    c0, _, g, _ = o.evaluate(flags)
    assert g.size == 7
    T0, ld0 = o.get_T_i_c(), o.get_line_delay()
    R = _qmat(T0[:4])

    def cost(T=T0, ld=ld0):
        o.set_T_i_c(T); o.set_line_delay(ld)
        c = o.evaluate(flags, residuals=False, gradient=False)[0]
        o.set_T_i_c(T0); o.set_line_delay(ld0)
        return c
    h = 1e-6
    for a in range(3):
        e = np.zeros(3); e[a] = h
        Tp, Tm = T0.copy(), T0.copy(); Tp[4:] += R @ e; Tm[4:] -= R @ e
        assert abs((cost(T=Tp) - cost(T=Tm)) / (2 * h) - g[a]) < 1e-6 * np.abs(g).max()
        Tp, Tm = T0.copy(), T0.copy(); Tp[:4] = _qmul(T0[:4], _qexp(e)); Tm[:4] = _qmul(T0[:4], _qexp(-e))
        assert abs((cost(T=Tp) - cost(T=Tm)) / (2 * h) - g[3 + a]) < 1e-6 * np.abs(g).max()
    hl = 1e-10
    assert abs((cost(ld=ld0 + hl) - cost(ld=ld0 - hl)) / (2 * hl) - g[6]) < 1e-5 * max(abs(g[6]), 1e-3 * np.abs(g).max())


# ---- CPU: API and CLI rules ----------------------------------------------------------------------------------------------------------
def test_reprojection_error_api_rules():
    from openimucameracalibrator_b200 import calibrator
    h = capi.CApi(calibrator.load_library(), "icc_", -1)             # host state: a host-only handle takes it
    h.set_reprojection_error("pixel"); h.set_reprojection_error(capi.REPROJ_ERROR_TANGENT)
    for bad in (2, -1):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
            h.set_reprojection_error(bad)
    ds = syn.make_dataset(syn.tiny_config())
    capi.load_dataset(h, ds, known_gravity=False)
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.set_reprojection_error("pixel")
    n = h.num_tangent(F_STAGE1)
    T = h.get_T_i_c()
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED.*CAM_INTRINSICS"):
        h.num_tangent(F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    assert h.num_tangent(F_STAGE1) == n and np.array_equal(h.get_T_i_c(), T)
    p = capi.CApi(calibrator.load_library(), "icc_", -1)              # the pixel residual keeps the extension flag
    capi.load_dataset(p, ds, known_gravity=False)
    assert p.num_tangent(F_STAGE1 | capi.FLAG_CAM_INTRINSICS) == n + len(ds["intrinsics"])


def test_reprojection_error_flag_is_parsed_and_checked(tmp_path):
    assert os.path.exists(HOT_CLI), "build the CLI first (__graft_entry__.build())"
    for bad in ("--reprojection_error=tangential", "--reprojection_error=Pixel", "--reprojection_error="):
        out = subprocess.run([HOT_CLI, bad], capture_output=True, text=True)
        assert out.returncode == 1 and "--reprojection_error must be 'pixel' or 'tangent'" in out.stderr, (bad, out.stderr)
    ds = syn.make_dataset(syn.tiny_config())
    paths = iof.write_dataset_files(ds, str(tmp_path))
    base = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + ["--parse_only"]
    runs = [subprocess.run(base + extra, capture_output=True, text=True) for extra in ([], ["--reprojection_error=pixel"], ["--reprojection_error", "tangent"])]
    assert all(r.returncode == 0 for r in runs), [r.stderr for r in runs]


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------------
def tangent_gpu(gpu_factory, ds, shard=None):
    g = gpu_factory(); g.set_reprojection_error("tangent"); capi.load_dataset(g, ds, shard=shard)
    return g


GPU_FLAGS = [F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_TIME_OFFSET | capi.FLAG_IMU_BIASES | capi.FLAG_GRAVITY_DIR,
             capi.FLAG_SPLINE | capi.FLAG_POINTS | capi.FLAG_CAM_LINE_DELAY]


@pytest.fixture(params=["tmem_always", "legacy"])
def vision_path(request, monkeypatch):
    """the persistent Jacobian kernel forced on, or the one-warp kernels forced on"""
    monkeypatch.delenv("ICC_TMEM_ALWAYS", raising=False); monkeypatch.delenv("ICC_VISION_LEGACY", raising=False)
    monkeypatch.setenv("ICC_TMEM_ALWAYS" if request.param == "tmem_always" else "ICC_VISION_LEGACY", "1")
    return request.param


def _parity(g, o, flags):
    cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
    co, ro, go, Ho = o.evaluate(flags, hessian=True)
    assert abs(cg - co) <= 1e-9 * abs(co), (cg, co)
    assert rel(rg, ro) < 1e-9 and rel(gg, go) < 1e-9 and rel(Hg, Ho) < 1e-9, (rel(rg, ro), rel(gg, go), rel(Hg, Ho))
    assert_scaled_parity(g, flags, (co, ro, go, Ho), (cg, rg, gg, Hg))


@pytest.mark.gpu
@pytest.mark.parametrize("model,k", CASES, ids=ALL_IDS)
def test_gpu_tangent_evaluation_matches_oracle(gpu_factory, vision_path, model, k):
    ds = syn.make_dataset(syn.tiny_config(model, k))
    g, o = tangent_gpu(gpu_factory, ds), tangent_oracle(ds)
    for flags in GPU_FLAGS:
        _parity(g, o, flags)
    gs = syn.make_dataset(syn.tiny_config(model, k, line_delay_truth=0.0))    # global shutter: the vision residuals keep zero weight
    gs["init_line_delay_s"] = 0.0
    _parity(tangent_gpu(gpu_factory, gs), tangent_oracle(gs), F_STAGE1)


@pytest.mark.gpu
def test_gpu_tangent_intrinsics_flag_is_refused_and_state_kept(gpu_factory):
    ds = syn.make_dataset(syn.tiny_config())
    g = tangent_gpu(gpu_factory, ds)
    T, kn = g.get_T_i_c(), g.get_knots()
    with pytest.raises(capi.IccError, match="ICC_ERR_UNSUPPORTED"):
        g.optimize(5, F_STAGE1 | capi.FLAG_CAM_INTRINSICS)
    assert np.array_equal(g.get_T_i_c(), T) and all(np.array_equal(a, b) for a, b in zip(g.get_knots(), kn))
    g.optimize(2, F_STAGE1)


def _two_stage_parity(g, o, ds):
    g1, o1 = g.optimize(50, F_STAGE1), o.optimize(50, F_STAGE1)
    assert (g1.iterations, g1.successful_steps, g1.termination) == (o1.iterations, o1.successful_steps, o1.termination)
    assert abs(g1.mean_reproj_error - pixel_mean_reproj(o, ds)) <= 1e-8 * g1.mean_reproj_error     # the product reports pixels
    g2, o2 = g.optimize(10, F_STAGE2), o.optimize(10, F_STAGE2)
    assert (g2.iterations, g2.successful_steps, g2.termination) == (o2.iterations, o2.successful_steps, o2.termination)
    assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8
    assert abs(g.get_line_delay() - o.get_line_delay()) <= 1e-7 * abs(o.get_line_delay())
    return g1, g2


@pytest.mark.gpu
def test_gpu_tangent_two_stage_lm_matches_oracle_small(gpu_factory):
    model, k = syn.CONFIGS[3].model, syn.CONFIGS[3].intrinsics
    ds = syn.make_dataset(syn.tiny_config(model, k, n_frames=60, line_delay_init_scale=1.1))
    _two_stage_parity(tangent_gpu(gpu_factory, ds), tangent_oracle(ds), ds)


@pytest.mark.gpu
def test_gpu_tangent_two_stage_lm_matches_oracle_config4(gpu_factory):
    ds = syn.make_dataset(syn.CONFIGS[4])
    g1, _ = _two_stage_parity(tangent_gpu(gpu_factory, ds), tangent_oracle(ds), ds)
    assert 0.15 < g1.mean_reproj_error < 0.4


@pytest.mark.gpu
def test_gpu_default_is_unchanged_by_an_explicit_pixel_mode(gpu_factory):
    """Per-corner residuals are bit-identical; the sums the kernels reduce with atomics (cost, J^T r, J^T J) differ between any two runs in
    the last bits, so those are held to the scatter of two default handles."""
    ds = syn.make_dataset(syn.tiny_config(cm.DOUBLE_SPHERE, syn.CONFIGS[3].intrinsics))
    a, a2 = gpu_factory(), gpu_factory(); capi.load_dataset(a, ds); capi.load_dataset(a2, ds)
    b = gpu_factory(); b.set_reprojection_error("pixel"); capi.load_dataset(b, ds)
    ea, ea2, eb = (h.evaluate(F_STAGE1, hessian=True) for h in (a, a2, b))
    assert np.array_equal(ea[1], eb[1])
    for i in (0, 2, 3):
        assert rel(np.atleast_1d(eb[i]), np.atleast_1d(ea[i])) <= max(4 * rel(np.atleast_1d(ea2[i]), np.atleast_1d(ea[i])), 1e-14)
    sa, sb = a.optimize(20, F_STAGE1), b.optimize(20, F_STAGE1)
    assert sa.iterations == sb.iterations and abs(sa.final_cost - sb.final_cost) <= 1e-12 * sa.final_cost
    assert rel(a.get_T_i_c(), b.get_T_i_c()) < 1e-12
    t = tangent_gpu(gpu_factory, ds)
    assert t.evaluate(F_STAGE1)[0] != ea[0]


def wide_dataset(tilt_deg=88.0, n_frames=40, seed=5):
    """A noise-free DoubleSphere sequence of the tiny configuration, with the camera tilted `tilt_deg` away from the board: every corner lies
    70-110 degrees off the optical axis, many of them past 90.  Built the way synthetic.make_dataset builds its sequences."""
    model, k = WIDE[0]
    cfg = syn.tiny_config(model, k, n_frames=n_frames, grid=(8, 6), seed=seed, corner_noise_px=0.0, imu_noise=False, square_m=0.05,
                          pose_noise_m=0.0, pose_noise_rad=0.0)
    ds = syn.make_dataset(cfg)
    tilt = syn.so3_exp(np.radians(tilt_deg) * np.array([1.0, 0.0, 0.0]))
    # the same IMU trajectory and streams; the camera (T_i_c) is rotated by `tilt`: re-observe every corner at its row time
    rng = np.random.default_rng(cfg.seed)
    q_ic, t_ic = ds["truth"]["T_i_c"][:4], ds["truth"]["T_i_c"][4:]
    R_ic = syn.quat_xyzw_to_matrix(q_ic)
    R_wc_base = np.diag([1.0, -1.0, -1.0]); p_wc_base = np.array([0.0, 0.0, 0.5])
    R_wi_base = R_wc_base @ R_ic.T; p_wi_base = p_wc_base - R_wi_base @ t_ic
    traj = syn.Trajectory(rng, R_wi_base, p_wi_base)
    R_ic2 = R_ic @ tilt
    X = ds["board_xyzw"][:, :3]; C = X.shape[0]; ld = ds["truth"]["line_delay"]
    y_row = np.full((n_frames, C), H / 2.0)
    for _ in range(30):
        t_obs = ds["frame_t"][:, None] + y_row * ld * cfg.dt_so3_s
        R = traj.R_wi(t_obs.ravel()).reshape(n_frames, C, 3, 3); p = traj.p_wi(t_obs.ravel()).reshape(n_frames, C, 3)
        pcam = np.einsum("ji,fcj->fci", R_ic2, np.einsum("fcji,fcj->fci", R, X[None] - p) - t_ic)
        uv, valid = cm.project(model, k, pcam)
        y_row = uv[..., 1]
    assert valid.all()
    ang = np.degrees(np.arccos(pcam[..., 2] / np.linalg.norm(pcam, axis=-1)))
    R_wc = traj.R_wi(ds["frame_t"]) @ R_ic2
    p_wc = traj.p_wi(ds["frame_t"]) + traj.R_wi(ds["frame_t"]) @ t_ic
    T_init = ds["T_i_c_init"].copy(); T_init[:4] = syn.matrix_to_quat_xyzw((syn.quat_xyzw_to_matrix(T_init[:4]) @ tilt)[None])[0]
    q2 = syn.matrix_to_quat_xyzw(R_ic2[None])[0]
    return dict(ds, uv=uv.reshape(-1, 2).copy(), q_wc=syn.matrix_to_quat_xyzw(R_wc), p_wc=p_wc, T_i_c_init=T_init, std_so3=1e-3, std_r3=1e-2,
                truth=dict(ds["truth"], T_i_c=np.concatenate([q2, t_ic]))), ang.ravel()


@pytest.mark.gpu
def test_gpu_tangent_wide_lens_past_90_degrees(gpu_factory):
    ds, ang = wide_dataset()
    assert (ang > 90.0).sum() > 0.2 * ang.size and ang.max() < 115.0
    g = tangent_gpu(gpu_factory, ds)
    o = tangent_oracle(ds)
    _parity(g, o, F_STAGE1)
    # corners past 90 degrees pull on the solution: nonzero, finite residuals and Jacobian rows
    r = g.evaluate(F_STAGE1)[1][: 2 * ang.size].reshape(-1, 2)
    far = ang > 90.0
    assert np.isfinite(r).all() and (np.abs(r[far]) < 1e3).all()
    qt, ld_t = ds["truth"]["T_i_c"], ds["truth"]["line_delay"]
    rot_err = lambda q: np.degrees(2 * np.arccos(min(1.0, abs(float(q[:4] @ qt[:4])))))   # noqa: E731
    e0 = rot_err(g.get_T_i_c())
    s1 = g.optimize(50, F_STAGE1); s2 = g.optimize(10, F_STAGE2)
    T = g.get_T_i_c()
    print(f"\n[tangent wide] start {e0:.3f} deg -> {rot_err(T):.2e} deg, |dt| {np.linalg.norm(T[4:] - qt[4:]):.2e} m, "
          f"line delay {g.get_line_delay():.6e} (truth {ld_t:.6e}), pixel error {s1.mean_reproj_error:.3e} px after stage 1, {g.mean_reprojection_error():.3e} px after stage 2")
    # noise-free corners, but a trajectory that no quintic B-spline holds exactly: the solve ends a few micro-pixels from zero
    assert rot_err(T) < 1e-3 and np.linalg.norm(T[4:] - qt[4:]) < 1e-6
    assert abs(g.get_line_delay() - ld_t) < 1e-4 * ld_t
    assert g.mean_reprojection_error() < 1e-4


@pytest.mark.gpu
def test_gpu_tangent_cli_chain(tmp_path):
    ds, ang = wide_dataset(n_frames=30)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    pj = str(tmp_path / "poses_tangent.json")
    r = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + paths["camera_calibration_json"],
                        "--output_pose_dataset=" + pj, "--pose_error", "tangent"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    out = {}
    for mode in ("pixel", "tangent"):
        rj = str(tmp_path / f"result_{mode}.json")
        args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items() if a not in ("input_pose_dataset", "result_output_json")]
        args += ["--input_pose_dataset=" + pj, "--result_output_json=" + rj, "--reprojection_error=" + mode, "--calibrate_cam_line_delay"]
        r = subprocess.run(args, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr + r.stdout
        out[mode] = json.load(open(rj))
    assert set(out["pixel"]) == set(out["tangent"])
    assert np.isfinite(out["tangent"]["final_reproj_error"])


@pytest.mark.gpu
def test_gpu_tangent_shards_are_additive(gpu_factory):
    """each shard forms the bearings of its own corners: the shards' sums equal the unsharded evaluation"""
    ds = syn.make_dataset(syn.tiny_config(cm.DOUBLE_SPHERE, syn.CONFIGS[3].intrinsics, n_frames=60))
    g = tangent_gpu(gpu_factory, ds)
    c, _, grad, _ = g.evaluate(F_STAGE1, residuals=False)
    cs, gs = 0.0, 0.0
    for rnk in range(2):
        s = tangent_gpu(gpu_factory, ds, shard=(rnk, 2))
        ci, _, gi, _ = s.evaluate(F_STAGE1, residuals=False)
        cs += ci; gs = gs + gi
    assert abs(cs - c) <= 1e-11 * c and rel(gs, grad) < 1e-10
