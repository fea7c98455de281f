"""The spline residual kernels outside the motion envelope of `synthetic.make_dataset`: a camera spinning about its optical axis at
12-48 rad/s (SO(3) knot increments up to 2.4 rad, so that sincos_small leaves its polynomials for the library sincos), motionless
lead-ins (repeated knots: zero increments, the series branches of so3_log / so3_jr_inv and the 1/theta guard of the increment
staging), large lever-arm and centripetal IMU terms, and arbitrary world frames.  The CPU tests check the generator and the oracle in
this regime; the GPU tests hold the kernels to the oracle at 1e-9, and every one of them first asserts through the branch census
that its data takes the branches it is about."""
import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, TangentWalker, qexp, qmul, rel
from motion_support import R_IC, branch_census, make_motion_dataset, truth_knots, world_tangent_map, world_transform_state
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_scaled_parity

TOL = 1e-9
INCREMENT = 2.4                      # rad per SO(3) knot interval at full spin: |lambda theta / 2| reaches 1.2 > pi/4
SPACINGS = ((0.05, 0.05), (0.1, 0.1), (0.15, 0.15), (0.2, 0.2), (0.07, 0.11))
WIDE = F_STAGE1 | capi.FLAG_CAM_INTRINSICS | capi.FLAG_TIME_OFFSET | capi.FLAG_IMU_INTRINSICS
FLAG_SETS = (F_STAGE1, F_ALL, F_STAGE1 | capi.FLAG_GRAVITY_DIR, WIDE)
MODELS = {cm.MODEL_NAMES[m].lower(): (m, i) for m, i in syn._CFG5_MODELS}   # the six distinct camera models of config 5


def fast_spin(dt=(0.05, 0.05), model=cm.FISHEYE, intrinsics=None, **kw):
    """Ramp from rest to the spin rate that makes one SO(3) knot interval INCREMENT rad."""
    if intrinsics is None:
        intrinsics = dict(syn._CFG5_MODELS)[model]
    kw.setdefault("spin_rate", INCREMENT / dt[0])
    return make_motion_dataset(model=model, intrinsics=intrinsics, dt_so3_s=dt[0], dt_r3_s=dt[1], **kw)


def static_lead_in(**kw):
    """0.5 s motionless in the world frame of the motionless IMU pose (its orientation is exactly the identity quaternion, so the
    repeated knots have exactly zero increments however the quaternion product is rounded), then a ramp to 16 rad/s."""
    return make_motion_dataset(n_frames=40, static_s=0.5, ramp_s=0.4, spin_rate=16.0, dt_so3_s=0.15, dt_r3_s=0.15, identity_start=True, **kw)


def _load(factory, ds, known_gravity=True):
    api = factory()
    capi.load_dataset(api, ds, known_gravity=known_gravity)
    truth_knots(api, ds)
    return api


# ---- CPU: the generator and the oracle in this regime -----------------------------------------------------------------------------

def test_generator_gyro_matches_rotation_differences():
    ds = fast_spin(imu_noise=False, static_s=0.2)
    R, om = ds["truth"]["R_wi"], ds["truth"]["omega"]
    t = np.linspace(-0.1, 0.9, 401)
    h = 1e-5
    Ra, Rb = R(t - h / 2), R(t + h / 2)
    fd = _log_batch(np.einsum("nji,njk->nik", Ra, Rb)) / h             # log(R(t - h/2)^T R(t + h/2)) / h = omega(t) + O(h^2)
    w = om(t)
    assert np.abs(w).max() > 40.0                                      # the spin reaches 48 rad/s
    assert np.abs(fd - w).max() < 1e-6 * np.abs(w).max()
    assert np.array_equal(w[t < 0.2], np.zeros_like(w[t < 0.2]))      # motionless lead-in: exactly zero rate
    gyr_true = ds["gyro"] - ds["gyr_bias"]
    t_imu = ds["imu_t"] + ds["time_offset_imu_to_cam_s"]
    assert np.abs(gyr_true - om(t_imu)).max() < 1e-12
    # the body rate is the spin about the optical axis (the camera's z axis in the IMU frame) plus the wobble
    late = t_imu > 0.6
    assert np.abs(gyr_true[late] @ R_IC[:, 2] - INCREMENT / 0.05).max() < 0.2 * INCREMENT / 0.05


def _log_batch(R):
    cos = np.clip((np.trace(R, axis1=1, axis2=2) - 1) / 2, -1, 1)
    th = np.arccos(cos)
    v = np.stack([R[:, 2, 1] - R[:, 1, 2], R[:, 0, 2] - R[:, 2, 0], R[:, 1, 0] - R[:, 0, 1]], -1)
    f = np.where(th < 1e-12, 0.5, th / (2 * np.sin(np.maximum(th, 1e-300))))
    return f[:, None] * v


def test_generator_corners_reproject_at_truth():
    """The noise-free corners are the fixed point of the reference's rolling-shutter model: projected at the truth pose of the times
    their own rows give, with the row offsets of the rotation and of the position taken on their own knot spacings."""
    for kw in (dict(dt=(0.07, 0.11)), dict(dt=(0.05, 0.05), model=cm.DOUBLE_SPHERE)):
        ds = fast_spin(**kw)
        T = ds["truth"]
        uv = T["uv"].reshape(len(ds["frame_t"]), -1, 2)
        y = uv[..., 1]
        tR = ds["frame_t"][:, None] + y * T["line_delay"] * ds["dt_so3_s"]
        tp = ds["frame_t"][:, None] + y * T["line_delay"] * ds["dt_r3_s"]
        R = T["R_wi"](tR.ravel()).reshape(uv.shape[:2] + (3, 3)); p = T["p_wi"](tp.ravel()).reshape(uv.shape[:2] + (3,))
        X = ds["board_xyzw"][:, :3]
        pc = np.einsum("ji,fcj->fci", R_IC, np.einsum("fcji,fcj->fci", R, X[None] - p) - T["T_i_c"][4:])
        uv2, ok = cm.project(ds["model"], ds["intrinsics"], pc)
        assert ok.all() and np.abs(uv2 - uv).max() < 1e-6
        assert np.abs(ds["uv"] - T["uv"]).max() < 2.0                 # 0.2 px noise


@pytest.mark.parametrize("which", ["fast_spin", "static_lead_in"])
def test_oracle_gradient_matches_central_differences(oracle_factory, which):
    ds = fast_spin(n_frames=16) if which == "fast_spin" else static_lead_in()
    o = _load(oracle_factory, ds, known_gravity=False)
    _, _, g, _ = o.evaluate(F_ALL)
    w = TangentWalker(o, F_ALL)
    rng = np.random.default_rng(3)
    nld = o.num_tangent(F_ALL & ~capi.FLAG_IMU_BIASES) - 1                  # the line-delay column: a proportionally smaller probe
    for _ in range(3):
        d = rng.normal(size=w.n); d[nld] *= 1e-4
        eps = 1e-7
        fd = (w.cost(eps * d) - w.cost(-eps * d)) / (2 * eps)
        assert abs(fd - g @ d) <= 2e-6 * max(abs(fd), abs(g @ d)), (fd, g @ d)
    w.restore()


def test_oracle_lm_recovers_truth_on_noise_free_fast_spin(oracle_factory):
    """With exact corners and IMU readings the only misfit left is the spline's approximation of the motion: the oracle's LM walks T_i_c
    from its 1 degree / 2 cm start to the truth, so the generator's corners, specific forces and rates describe one motion."""
    ds = fast_spin(dt=(0.05, 0.05), spin_rate=12.0, corner_noise_px=0.0, imu_noise=False, n_frames=30)
    o = _load(oracle_factory, ds)
    T0 = o.get_T_i_c()
    s = o.optimize(50, F_STAGE1)
    T = o.get_T_i_c(); Tt = ds["truth"]["T_i_c"]
    ang = lambda a, b: 2 * np.arcsin(min(1.0, np.linalg.norm(qmul(a[:4] * [-1, -1, -1, 1], b[:4])[:3])))   # noqa: E731
    assert ang(T0, Tt) > 0.015 and s.termination != 4
    assert ang(T, Tt) < 1e-4 and np.linalg.norm(T[4:] - Tt[4:]) < 1e-4, (ang(T, Tt), T[4:] - Tt[4:])


def test_census_reaches_every_branch(oracle_factory):
    """The datasets of the GPU tests take the branches those tests are about (checked here too, so that a generator change shows up
    without a GPU)."""
    for dt in SPACINGS:
        ds = fast_spin(dt=dt)
        c = branch_census(_load(oracle_factory, ds), ds)
        assert c["vision"]["library_sincos"] > 0 and c["imu"]["library_sincos"] > 0 and c["max_increment_rad"] < 2.6
    ds = static_lead_in()
    c = branch_census(_load(oracle_factory, ds), ds)
    for tag in ("vision", "imu"):
        assert c[tag]["theta_zero"] > 0 and c[tag]["jr_series"] > 0 and c[tag]["library_sincos"] > 0 and c[tag]["closed_form"] > 0


# ---- GPU ----------------------------------------------------------------------------------------------------------------------------

def _assert_eval_parity(o, g, flags):
    co, ro, go, Ho = o.evaluate(flags, hessian=True)
    cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
    assert np.isfinite(cg) and np.isfinite(rg).all() and np.isfinite(gg).all() and np.isfinite(Hg).all()
    assert abs(cg - co) <= TOL * abs(co)
    assert rel(rg, ro) < TOL and rel(gg, go) < TOL and rel(Hg, Ho) < TOL
    assert_scaled_parity(g, flags, (co, ro, go, Ho), (cg, rg, gg, Hg))
    c2 = g.evaluate(flags, residuals=False, gradient=False)[0]
    assert abs(c2 - cg) <= 1e-12 * abs(cg)
    return rg


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_eval_parity_fast_spin(oracle_factory, gpu_factory, eval_path, name):
    model, intr = MODELS[name]
    for dt in SPACINGS:
        ds = fast_spin(dt=dt, model=model, intrinsics=intr)
        o, g = _load(oracle_factory, ds, known_gravity=False), _load(gpu_factory, ds, known_gravity=False)
        c = branch_census(g, ds)
        assert c["vision"]["library_sincos"] > 0 and c["imu"]["library_sincos"] > 0, c
        for flags in FLAG_SETS:
            r = _assert_eval_parity(o, g, flags)
            assert not (r == 1e10).any()


def _edge_knots(api, ds, first, edges, rng):
    """SO(3) knots with the increments `edges` (rad) from knot `first` on, about axes near the optical axis (the board stays in view);
    the knots before `first` are the truth's and the increments after the edges repeat the truth's, so every increment stays below pi."""
    so3, r3, ba, bg = api.get_knots()
    inc = [qmul(so3[i] * [-1, -1, -1, 1], so3[i + 1]) for i in range(len(so3) - 1)]
    a = R_IC[:, 2]
    for j, th in enumerate(edges):
        ax = a + 0.05 * rng.normal(size=3); ax /= np.linalg.norm(ax)
        inc[first + j] = qexp(th * ax)
    q = so3.copy()
    for i in range(first, len(so3) - 1):
        q[i + 1] = qmul(q[i], inc[i])
    return q


EDGES = (0.0, 1e-12, 1e-8, 1e-4, 1.0, 2.0, 2.8)


@pytest.mark.gpu
def test_knot_edges_through_set_knots(oracle_factory, gpu_factory, eval_path):
    ds = fast_spin(dt=(0.05, 0.05), spin_rate=20.0, n_frames=30)
    o, g = _load(oracle_factory, ds, known_gravity=False), _load(gpu_factory, ds, known_gravity=False)
    q = _edge_knots(g, ds, 6, EDGES, np.random.default_rng(4))
    for api in (o, g):
        api.set_knots(q, None, None, None)
    c = branch_census(g, ds)
    for tag in ("vision", "imu"):
        assert min(c[tag][k] for k in ("library_sincos", "theta_zero", "log_series", "jr_series")) > 0, c
    for flags in (F_STAGE1, F_ALL):
        r = _assert_eval_parity(o, g, flags)
        assert not (r == 1e10).any()
    flags = F_STAGE1 | capi.FLAG_GRAVITY_DIR | capi.FLAG_IMU_BIASES
    grad = g.evaluate(flags)[2]
    w = TangentWalker(g, flags)
    rng = np.random.default_rng(1)
    for _ in range(3):
        d = rng.normal(size=w.n); eps = 1e-7
        fd = (w.cost(eps * d) - w.cost(-eps * d)) / (2 * eps)
        assert np.isfinite(fd) and abs(fd - grad @ d) <= 2e-6 * abs(fd)
    w.restore()


@pytest.mark.gpu
def test_static_lead_in_eval_parity(oracle_factory, gpu_factory, eval_path):
    ds = static_lead_in()
    o, g = _load(oracle_factory, ds, known_gravity=False), _load(gpu_factory, ds, known_gravity=False)
    so3 = g.get_knots()[0]
    assert np.array_equal(so3[0], [0.0, 0.0, 0.0, 1.0]) and np.array_equal(so3[1], so3[0])
    c = branch_census(g, ds)
    for tag in ("vision", "imu"):
        assert c[tag]["theta_zero"] > 0 and c[tag]["library_sincos"] > 0, c
    for flags in FLAG_SETS:
        _assert_eval_parity(o, g, flags)


@pytest.mark.gpu
def test_world_frame_equivariance(gpu_factory):
    """A rigid change of world frame x' = G x + t leaves cost and residuals unchanged and maps J^T r and J^T J by P (GPU alone)."""
    rng = np.random.default_rng(8)
    frames = [(np.diag([1.0, -1.0, -1.0]), np.zeros(3)), (np.diag([-1.0, 1.0, -1.0]), np.zeros(3)), (np.diag([-1.0, -1.0, 1.0]), np.zeros(3)),
              (syn.so3_exp(rng.normal(size=3)), np.zeros(3)), (syn.so3_exp(rng.normal(size=3)), rng.normal(size=3)),
              (np.eye(3), np.array([20.0, 0.0, 0.0]))]
    ds = fast_spin(dt=(0.1, 0.1))
    g0 = _load(gpu_factory, ds, known_gravity=False)
    c0, r0, gr0, H0 = g0.evaluate(F_ALL, hessian=True)
    assert branch_census(g0, ds)["vision"]["library_sincos"] > 0
    for G, t in frames:
        dsw = dict(ds); dsw["board_xyzw"] = np.concatenate([ds["board_xyzw"][:, :3] @ G.T + t, np.ones((len(ds["board_xyzw"]), 1))], -1)
        dsw["gravity"] = G @ ds["gravity"]
        g1 = gpu_factory(); capi.load_dataset(g1, dsw, known_gravity=False)
        world_transform_state(g0, g1, G, t)
        c1, r1, gr1, H1 = g1.evaluate(F_ALL, hessian=True)
        P = world_tangent_map(g0, F_ALL, G)
        assert abs(c1 - c0) <= 1e-10 * c0 and rel(r1, r0) < 1e-10
        assert rel(gr1, P @ gr0) < 1e-9 and rel(H1, P @ H0 @ P.T) < 1e-9


def _lm_two_stage(o, g):
    for flags, iters in ((F_STAGE1, 50), (F_STAGE2, 10)):
        so, sg = o.optimize(iters, flags), g.optimize(iters, flags)
        assert sg.iterations == so.iterations and sg.termination == so.termination and so.termination != 4
        assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8
        for a, b in zip(g.get_knots()[:2], o.get_knots()[:2]):
            assert rel(a, b) < 1e-8
    assert abs(g.get_line_delay() - o.get_line_delay()) <= 1e-8 * abs(o.get_line_delay())


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["fast_spin", "static_lead_in"])
def test_lm_parity_two_stage(oracle_factory, gpu_factory, which):
    ds = fast_spin(dt=(0.1, 0.1), n_frames=30) if which == "fast_spin" else static_lead_in()
    o, g = _load(oracle_factory, ds), _load(gpu_factory, ds)
    c = branch_census(g, ds)
    assert c["vision"]["library_sincos"] > 0 and c["imu"]["library_sincos"] > 0, c
    _lm_two_stage(o, g)


@pytest.mark.gpu
def test_eval_trajectory_fast_spin_on_knot_times(oracle_factory, gpu_factory):
    ds = fast_spin(dt=(0.05, 0.05))
    o, g = _load(oracle_factory, ds), _load(gpu_factory, ds)
    t_used = g.imu_used()[0]
    start_ns = int(ds["frame_t"][0] * 1e9)
    on_knots = start_ns + np.arange(g.num_knots()[0]) * int(ds["dt_so3_s"] * 1e9)
    t_ns = np.concatenate([(t_used * 1e9).astype(np.int64), on_knots.astype(np.int64), on_knots[1:-1].astype(np.int64) + 1])
    a, b = g.eval_trajectory(t_ns), o.eval_trajectory(t_ns)
    assert np.array_equal(a["valid"], b["valid"]) and a["valid"][len(t_used):].sum() > 5
    assert np.abs(a["gyro"][a["valid"] == 1]).max() > 30.0
    for key in ("gyro", "accel", "gyro_bias", "accel_bias", "pose_q", "pose_p"):
        assert rel(a[key], b[key]) < TOL, key
