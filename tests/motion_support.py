"""Synthetic datasets outside the motion envelope of `synthetic.make_dataset`: a camera spinning about its own optical axis at up to
tens of rad/s, optional motionless lead-in, any world frame; and a census of which SO(3) branches of the residual kernels the
observations of a loaded problem take.  NumPy only.

The dict returned by `make_motion_dataset` has `synthetic.make_dataset`'s keys, so `capi.load_dataset` takes it unchanged.  Its
`truth` entry also carries the trajectory as callables (`R_wi(t)`, `p_wi(t)`, camera clock) and the noise-free corners."""
from __future__ import annotations

import numpy as np

from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn

# thresholds of csrc/icc_device_math.cuh (kEps, the Taylor switch of so3_jr_inv / so3_exp_jr) and csrc/icc_vision_rows.cuh
# (sincos_small: fdlibm polynomials up to pi/4, library sincos beyond)
K_EPS = 1e-10
JR_SERIES_TH2 = 1e-6
SINCOS_POLY_MAX = 0.78539816339744828

# truth extrinsics of synthetic.make_dataset (README dataset 1)
_Q_IC = np.array([-0.007, -0.708, 0.706, 0.005]) / np.linalg.norm([-0.007, -0.708, 0.706, 0.005])
R_IC = syn.quat_xyzw_to_matrix(_Q_IC)
T_IC = np.array([0.007, -0.022, 0.001])


def _smoothstep(tau):
    """Quintic smoothstep S, S' and the integral of S from 0, for tau clipped to [0, 1] (C2 at both ends)."""
    c = np.clip(tau, 0.0, 1.0)
    S = c ** 3 * (10 - 15 * c + 6 * c * c)
    dS = 30 * c * c * (1 - c) ** 2
    iS = c ** 4 * (2.5 - 3 * c + c * c) + np.maximum(tau - 1.0, 0.0)
    return S, dS, iS


class SpinTrajectory:
    """R_wi(t) = R_b exp(alpha(t) a) exp(psi(t)), a = the optical axis in the IMU frame, psi = E(t) R_ic w(t) a small body-fixed wobble of the
    optical axis; p_wc(t) = p_c0 + E(t) s(t).  alpha' = rate * E(t), E a quintic ramp from 0 at `static_s` to 1 at `static_s + ramp_s`
    (a step at `static_s` when ramp_s = 0).  Before `static_s` rotation and position are exactly constant (bit for bit)."""

    def __init__(self, R_b, p_c0, rate, static_s, ramp_s, wobble_rad, wobble_hz, shift_m, rng):
        self.R_b, self.p_c0, self.rate, self.t0, self.T = R_b, p_c0, rate, static_s, ramp_s
        self.a = R_IC[:, 2].copy()
        self.w_amp = wobble_rad * rng.uniform(0.7, 1.0, size=2)
        self.w_f = wobble_hz * rng.uniform(0.8, 1.25, size=2)
        self.w_ph = rng.uniform(0, 2 * np.pi, size=2)
        self.s_amp = shift_m * rng.uniform(0.5, 1.0, size=3)
        self.s_f = rng.uniform(0.4, 1.2, size=3)
        self.s_ph = rng.uniform(0, 2 * np.pi, size=3)

    def _ramp(self, t):
        t = np.asarray(t, dtype=np.float64)
        if self.T == 0.0:
            on = (t >= self.t0).astype(np.float64)
            return on, np.zeros_like(t), np.maximum(t - self.t0, 0.0)
        S, dS, iS = _smoothstep((t - self.t0) / self.T)
        return S, dS / self.T, iS * self.T

    def _psi(self, t):
        """psi(t) and psi'(t) in the IMU frame."""
        t = np.asarray(t, dtype=np.float64)
        E, dE, _ = self._ramp(t)
        arg = 2 * np.pi * self.w_f * t[..., None] + self.w_ph
        w = np.concatenate([self.w_amp * np.sin(arg), np.zeros(t.shape + (1,))], -1)
        dw = np.concatenate([self.w_amp * 2 * np.pi * self.w_f * np.cos(arg), np.zeros(t.shape + (1,))], -1)
        psi_c = E[..., None] * w
        dpsi_c = dE[..., None] * w + E[..., None] * dw
        return psi_c @ R_IC.T, dpsi_c @ R_IC.T

    def alpha(self, t):
        E, _, iE = self._ramp(t)
        return self.rate * iE, self.rate * E

    def R_wi(self, t):
        al, _ = self.alpha(t)
        psi, _ = self._psi(t)
        return self.R_b @ syn.so3_exp(al[..., None] * self.a) @ syn.so3_exp(psi)

    def omega_body(self, t):
        """Analytic body rate: R^T R' = [exp(psi)^T alpha' a + Jr(psi) psi']x."""
        _, dal = self.alpha(t)
        psi, dpsi = self._psi(t)
        Ep = syn.so3_exp(psi)
        return np.einsum("...ji,j->...i", Ep, self.a) * dal[..., None] + (syn.so3_right_jacobian(psi) @ dpsi[..., None])[..., 0]

    def p_wc(self, t):
        t = np.asarray(t, dtype=np.float64)
        E, _, _ = self._ramp(t)
        s = self.s_amp * np.sin(2 * np.pi * self.s_f * t[..., None] + self.s_ph)
        return self.p_c0 + E[..., None] * s

    def p_wi(self, t):
        return self.p_wc(t) - self.R_wi(t) @ T_IC

    def acc_world(self, t, h=1e-3):
        """p_wi'' by the five-point stencil: truncation h^4/90 |p^(6)| < 1e-5 m/s^2 up to 50 rad/s, far below the accelerometer noise."""
        f = [self.p_wi(np.asarray(t) + k * h) for k in (-2, -1, 0, 1, 2)]
        return (-f[0] + 16 * f[1] - 30 * f[2] + 16 * f[3] - f[4]) / (12 * h * h)


def rot_x180():
    return np.diag([1.0, -1.0, -1.0])


def make_motion_dataset(model=cm.FISHEYE, intrinsics=(435.5, 1.0, 0.0, 479.1, 274.5, 0.05, 0.07, -0.11, 0.05), n_frames=24, fps=30.0,
                        grid=(6, 5), square_m=0.021, imu_rate_hz=200.0, seed=0, spin_rate=12.0, ramp_s=0.3, static_s=0.0,
                        wobble_rad=0.05, wobble_hz=1.0, shift_m=0.01, dt_so3_s=0.05, dt_r3_s=0.05, world_R=None, world_t=(0.0, 0.0, 0.0),
                        identity_start=False, corner_noise_px=0.2, imu_noise=True, tic_rot_perturb_rad=np.deg2rad(1.0),
                        time_offset_imu_to_cam_s=-0.0813, image_size=(960, 540)) -> dict:
    """Camera 0.5 m above the board looking straight at it, spinning about its optical axis.  The spin rate ramps from 0 (at
    `static_s`) to `spin_rate` rad/s over `ramp_s`; the first `static_s` seconds are motionless: identical frame poses (one pose prior
    repeated exactly) and IMU readings R^T g + bias (+ noise).  The world frame is (world_R, world_t) applied to the board-aligned frame
    (gravity +z there); `identity_start` instead picks the world frame in which the motionless IMU orientation is exactly the identity."""
    rng = np.random.default_rng(seed)
    W, H = image_size
    ld_true = 1.0 / fps / H
    cols, rows = grid
    gx, gy = np.meshgrid((np.arange(cols) - (cols - 1) / 2) * square_m, (np.arange(rows) - (rows - 1) / 2) * square_m)
    X0 = np.stack([gx.ravel(), gy.ravel(), np.zeros(cols * rows)], -1)
    C = X0.shape[0]
    R_wc_base = rot_x180()
    p_wc_base = np.array([0.0, 0.0, 0.5])
    R_wi_base = R_wc_base @ R_IC.T
    G = np.eye(3) if world_R is None else np.asarray(world_R, dtype=np.float64)
    if identity_start:
        G = R_wi_base.T.copy()
    tw = np.asarray(world_t, dtype=np.float64)
    R_b = np.eye(3) if identity_start else G @ R_wi_base
    traj = SpinTrajectory(R_b, G @ p_wc_base + tw, spin_rate, static_s, ramp_s, wobble_rad, wobble_hz, shift_m, rng)
    X = X0 @ G.T + tw
    gravity = G @ np.array([0.0, 0.0, 9.81])

    # rolling shutter, the reference's model: row y shifts the normalised times u_so3 and u_r3 by y * ld, i.e. the physical time by
    # y * ld * dt_so3 for the rotation and y * ld * dt_r3 for the position
    frame_t = np.arange(n_frames) / fps
    y_row = np.full((n_frames, C), H / 2.0)
    for _ in range(6):
        tR = frame_t[:, None] + y_row * ld_true * dt_so3_s
        tp = frame_t[:, None] + y_row * ld_true * dt_r3_s
        R = traj.R_wi(tR.ravel()).reshape(n_frames, C, 3, 3)
        p = traj.p_wi(tp.ravel()).reshape(n_frames, C, 3)
        q_imu = np.einsum("fcji,fcj->fci", R, X[None] - p)
        p_cam = np.einsum("ji,fcj->fci", R_IC, q_imu - T_IC)
        uv, valid = cm.project(model, intrinsics, p_cam)
        y_row = uv[..., 1]
    assert valid.all(), "motion dataset left the camera model's valid domain"
    uv_noisy = uv + rng.normal(0.0, corner_noise_px, size=uv.shape)

    # pose priors T_wc at the frame times; one noise draw repeated over the motionless frames
    R_wi_f = traj.R_wi(frame_t)
    R_wc = R_wi_f @ R_IC
    p_wc = traj.p_wc(frame_t)
    nR = rng.normal(0.0, np.deg2rad(0.2), size=(n_frames, 3)); nP = rng.normal(0.0, 2e-3, size=(n_frames, 3))
    still = frame_t + H * ld_true * max(dt_so3_s, dt_r3_s) < static_s
    nR[still] = nR[0]; nP[still] = nP[0]
    q_wc = syn.matrix_to_quat_xyzw(R_wc @ syn.so3_exp(nR))
    p_wc_n = p_wc + nP

    duration = frame_t[-1]
    n_imu = int(np.floor((duration + 0.5) * imu_rate_hz)) + 1
    t_cam = np.arange(n_imu) / imu_rate_hz - 0.25
    R_i = traj.R_wi(t_cam)
    acc = np.einsum("nji,nj->ni", R_i, traj.acc_world(t_cam) + gravity)
    gyr = traj.omega_body(t_cam)
    b_a = np.array([0.05, -0.03, 0.02]); b_g = np.array([2e-3, -1e-3, 5e-4])
    sig_a = 1.5e-2 * np.sqrt(imu_rate_hz); sig_g = 1.1e-3 * np.sqrt(imu_rate_hz)
    if imu_noise:
        acc = acc + rng.normal(0.0, sig_a, size=acc.shape)
        gyr = gyr + rng.normal(0.0, sig_g, size=gyr.shape)
    acc = acc + b_a
    gyr = gyr + b_g

    axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
    q_ic_init = syn.matrix_to_quat_xyzw(R_IC @ syn.so3_exp(axis * tic_rot_perturb_rad))
    return dict(
        name=f"spin_{cm.MODEL_NAMES[model].lower()}_{spin_rate:g}rads", model=model, intrinsics=np.asarray(intrinsics, dtype=np.float64),
        image_size=(W, H), fps=fps, board_xyzw=np.concatenate([X, np.ones((C, 1))], -1), frame_t=frame_t,
        corner_offsets=(np.arange(n_frames + 1) * C).astype(np.int32), point_ids=np.tile(np.arange(C, dtype=np.int32), n_frames),
        uv=uv_noisy.reshape(-1, 2).copy(), q_wc=q_wc, p_wc=p_wc_n, imu_t=t_cam - time_offset_imu_to_cam_s, accel=acc, gyro=gyr,
        dt_so3_s=dt_so3_s, dt_r3_s=dt_r3_s, std_so3=sig_g if imu_noise else 1.0, std_r3=sig_a if imu_noise else 1.0,
        time_offset_imu_to_cam_s=time_offset_imu_to_cam_s, init_line_delay_s=ld_true, T_i_c_init=np.concatenate([q_ic_init, np.zeros(3)]),
        acc_bias=b_a, gyr_bias=b_g, gravity=gravity,
        truth=dict(T_i_c=np.concatenate([_Q_IC, T_IC]), line_delay=ld_true, gravity=gravity, R_wi=traj.R_wi, p_wi=traj.p_wi,
                   omega=traj.omega_body, uv=uv.reshape(-1, 2).copy(), world_R=G, world_t=tw, traj=traj),
    )


# ---- spline state ---------------------------------------------------------------------------------------------------------------
# Knots are zero-based in time (quirk q7): knot j of a spline with spacing dt sits at start + (j - 2) dt in the sense that the order-6
# uniform B-spline reproduces a linear function (and a constant-rate rotation about a fixed axis) exactly from samples taken there.

def truth_knots(api, ds):
    """Set the problem's SO(3) / R^3 knots to the truth trajectory sampled at the knots' Greville times (a far better start than the
    reference's initialiser, whose knots lag the spline by two knot intervals, i.e. by radians at these rates)."""
    so3, r3, _, _ = api.get_knots()
    t0 = float(np.min(ds["frame_t"]))
    ts = t0 + (np.arange(len(so3)) - 2.0) * ds["dt_so3_s"]
    tr = t0 + (np.arange(len(r3)) - 2.0) * ds["dt_r3_s"]
    q = syn.matrix_to_quat_xyzw(ds["truth"]["R_wi"](ts))
    # consecutive knots on the same hemisphere, as the knot initialiser leaves them (the log takes the short way either way)
    for i in range(1, len(q)):
        if q[i] @ q[i - 1] < 0:
            q[i] = -q[i]
    api.set_knots(q, ds["truth"]["p_wi"](tr), None, None)


def cum_coeffs6(u):
    """Cumulative blending coefficients lambda_1..5(u) of the order-6 uniform B-spline (u may leave [0, 1) by the row time)."""
    u = np.asarray(u, dtype=np.float64)

    def N5(x):   # cardinal quintic B-spline on [0, 6]
        k = np.arange(7)
        binom = np.array([1, 6, 15, 20, 15, 6, 1], dtype=np.float64)
        return (((-1.0) ** k) * binom * np.maximum(x[..., None] - k, 0.0) ** 5).sum(-1) / 120.0

    B = np.stack([N5(u + 5 - j) for j in range(6)], -1)
    return np.cumsum(B[..., ::-1], -1)[..., ::-1][..., 1:]


def _qmul(a, b):
    ax, ay, az, aw = np.moveaxis(a, -1, 0); bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def _so3_log(q):
    """SO3::log with the branches of icc_device_math.cuh: -> (d, n2)."""
    n2 = (q[..., :3] ** 2).sum(-1)
    w = q[..., 3]
    n = np.sqrt(n2)
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(n2 < K_EPS * K_EPS, 2.0 / w - (2.0 / 3.0) * n2 / (w ** 3),
                     np.where(np.abs(w) < K_EPS, np.where(w > 0, np.pi, -np.pi) / n, 2.0 * np.arctan(n / w) / n))
    return f[..., None] * q[..., :3], n2


def _calc_times(t_s, start_ns, dt_s, n_knots):
    t_ns = (np.asarray(t_s) * 1e9).astype(np.int64)
    dt_ns = np.int64(dt_s * 1e9)
    st = t_ns - start_ns
    s = st // dt_ns
    ok = (st >= 0) & (s + 6 <= n_knots)
    return np.where(ok, s, 0), (st % dt_ns) / float(dt_ns), ok


BRANCHES = ("library_sincos", "theta_zero", "log_series", "jr_series", "closed_form")


def branch_census(api, ds):
    """For the problem loaded in `api` (its current knots, line delay and kept IMU samples), count the observations whose window takes each
    SO(3) branch of the kernels, separately for vision (one per corner) and IMU (one per kept sample).  An observation counts once per
    branch that any of its five increments takes:
      library_sincos  |lambda_i theta_i / 2| > pi/4 (sincos_small leaves its polynomials);
      theta_zero      the increment is exactly 0 (the 1/theta guard of the increment staging); counted from an unfused quaternion
                      product, the device's fused one leaves a ~1e-17 residue unless the products are exact (identity knots);
      log_series      |imag(R_i^-1 R_i+1)|^2 < kEps^2 (so3_log's series);
      jr_series       theta^2 < 1e-6 (the series of so3_jr_inv / so3_exp_jr);
      closed_form     theta^2 >= 1e-6."""
    so3 = api.get_knots()[0]
    d, n2 = _so3_log(_qmul(so3[:-1] * np.array([-1, -1, -1, 1.0]), so3[1:]))
    th = np.sqrt((d ** 2).sum(-1))
    start_ns = np.int64(float(np.min(ds["frame_t"])) * 1e9)
    ld = api.get_line_delay()
    # vision: per corner, u_so3 of its frame plus row * line delay, segment of the frame
    off = ds["corner_offsets"]
    s_f, u_f, ok_f = _calc_times(ds["frame_t"], start_ns, ds["dt_so3_s"], len(so3))
    _, _, ok_r = _calc_times(ds["frame_t"], start_ns, ds["dt_r3_s"], len(api.get_knots()[1]))
    fr = np.repeat(np.arange(len(ds["frame_t"])), np.diff(off))
    keep = (ok_f & ok_r)[fr]
    vis = (s_f[fr][keep], u_f[fr][keep] + np.asarray(ds["uv"])[keep, 1] * ld)
    t_imu = api.imu_used()[0]
    s_i, u_i, ok_i = _calc_times(t_imu, start_ns, ds["dt_so3_s"], len(so3))
    imu = (s_i[ok_i], u_i[ok_i])
    out = {}
    for tag, (s, u) in (("vision", vis), ("imu", imu)):
        idx = s[:, None] + np.arange(5)
        lam = cum_coeffs6(u)
        x = 0.5 * lam * th[idx]
        t2 = th[idx] ** 2
        out[tag] = dict(observations=int(len(s)), library_sincos=int((np.abs(x) > SINCOS_POLY_MAX).any(-1).sum()),
                        theta_zero=int((th[idx] == 0.0).any(-1).sum()), log_series=int((n2[idx] < K_EPS * K_EPS).any(-1).sum()),
                        jr_series=int((t2 < JR_SERIES_TH2).any(-1).sum()), closed_form=int((t2 >= JR_SERIES_TH2).any(-1).sum()))
    out["max_increment_rad"] = float(th.max())
    return out


def world_transform_state(api_src, api_dst, G, t):
    """Copy the spline state of `api_src` into `api_dst` expressed in the world frame x' = G x + t: SO(3) knots G R, R^3 knots G p + t,
    gravity G g; T_i_c, biases and line delay are body quantities and stay."""
    so3, r3, ba, bg = api_src.get_knots()
    qG = syn.matrix_to_quat_xyzw(G)
    api_dst.set_knots(_qmul(np.broadcast_to(qG, so3.shape), so3), r3 @ G.T + t, ba, bg)
    api_dst.set_T_i_c(api_src.get_T_i_c())
    api_dst.set_line_delay(api_src.get_line_delay())
    api_dst.set_known_gravity_dir(G @ api_src.get_gravity())


def world_tangent_map(api, flags, G):
    """P of the tangent space under x' = G x + t (canonical order): identity on SO(3) knots (right increments), T_i_c, line delay and
    biases; G on each R^3 knot and on gravity."""
    from openimucameracalibrator_b200 import _capi as capi
    n = api.num_tangent(flags)
    nso3, nr3, _, _ = api.num_knots()
    P = np.eye(n)
    off = 0
    if flags & capi.FLAG_SPLINE:
        off += 3 * nso3
        for i in range(nr3):
            P[off + 3 * i: off + 3 * i + 3, off + 3 * i: off + 3 * i + 3] = G
        off += 3 * nr3
    if flags & capi.FLAG_T_I_C:
        off += 6
    if flags & capi.FLAG_GRAVITY_DIR:
        P[off: off + 3, off: off + 3] = G
    return P
