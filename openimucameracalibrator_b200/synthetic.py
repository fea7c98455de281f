"""Deterministic synthetic board + IMU sequences for the BASELINE.json configurations (SURVEY.md §8(d)).

Everything the hot CLI reads from files (continuous_time_imu_to_camera_calibration.cc:91-199) is produced here as
arrays: board points, per-frame corner observations (rolling-shutter, the reference's own row-time model — SURVEY quirk
q2: row time `y * line_delay` is added to the *normalised* knot time), per-frame PnP-like pose priors, IMU streams with
bias + noise, spline weighting, initial T_i_c.  The same arrays drive the CUDA solver, the CPU oracle and the file
writers in `io_formats.py`.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from . import camera_models as cm


@dataclass
class SyntheticConfig:
    name: str
    model: int
    intrinsics: tuple
    n_frames: int
    grid: tuple            # (cols, rows) -> C = cols*rows corners
    imu_rate_hz: float
    seed: int
    fps: float = 30.0
    image_size: tuple = (960, 540)
    dt_so3_s: float = 0.05
    dt_r3_s: float = 0.05
    square_m: float = 0.021
    line_delay_truth: float = field(default=None)   # default 1/fps/height (app :186)
    line_delay_init_scale: float = 1.0
    time_offset_imu_to_cam_s: float = -0.0813
    corner_noise_px: float = 0.2
    pose_noise_m: float = 2e-3
    pose_noise_rad: float = np.deg2rad(0.2)
    tic_rot_perturb_rad: float = np.deg2rad(1.0)
    imu_noise: bool = True


# Truth intrinsics from the reference's README tables (Readme.md:31-39), Theia parameter order.
_F, _CX, _CY = 437.1, 489.1, 270.9
CONFIGS = {
    1: SyntheticConfig("cfg1_division_undistortion_60x35", cm.DIVISION_UNDISTORTION, (437.1, 1.0, 489.1, 270.9, -1.44e-6), 60, (7, 5), 200.0, 1235),
    2: SyntheticConfig("cfg2_fisheye_300x96", cm.FISHEYE, (435.5, 1.0, 0.0, 479.1, 274.5, 0.05, 0.07, -0.11, 0.05), 300, (12, 8), 200.0, 1236),
    3: SyntheticConfig("cfg3_double_sphere_rs_1000x96", cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513), 1000, (12, 8), 400.0, 1237,
                       line_delay_init_scale=1.1),
    4: SyntheticConfig("cfg4_extended_unified_3000x144", cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062), 3000, (16, 9), 1000.0, 1238),
}
# config 5: eight independent config-2-shaped sequences, models cycling (SURVEY §8(d))
_CFG5_MODELS = [
    (cm.PINHOLE, (437.0, 1.0, 0.0, 489.0, 271.0, -0.05, 0.01)),
    (cm.FISHEYE, (435.5, 1.0, 0.0, 479.1, 274.5, 0.05, 0.07, -0.11, 0.05)),
    (cm.DIVISION_UNDISTORTION, (437.1, 1.0, 489.1, 270.9, -1.44e-6)),
    (cm.DOUBLE_SPHERE, (342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513)),
    (cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062)),
    (cm.FOV, (437.0, 1.0, 489.0, 271.0, 0.9)),
    (cm.FISHEYE, (435.5, 1.0, 0.0, 479.1, 274.5, 0.05, 0.07, -0.11, 0.05)),
    (cm.EXTENDED_UNIFIED, (438.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062)),
]


def config5(k: int) -> SyntheticConfig:
    model, intr = _CFG5_MODELS[k % 8]
    return SyntheticConfig(f"cfg5_seq{k}_{cm.MODEL_NAMES[model].lower()}_300x96", model, intr, 300, (12, 8), 200.0, 1234 + 10 * k)


def tiny_config(model: int = cm.DIVISION_UNDISTORTION, intr=(437.1, 1.0, 489.1, 270.9, -1.44e-6), n_frames: int = 24,
                grid=(5, 4), imu_rate_hz: float = 100.0, seed: int = 7, **kw) -> SyntheticConfig:
    return SyntheticConfig(f"tiny_{cm.MODEL_NAMES[model].lower()}", model, tuple(intr), n_frames, grid, imu_rate_hz, seed, **kw)


# ---- small SO(3) helpers (numpy, batch) --------------------------------------------------------------------------

def _hat(v):
    z = np.zeros_like(v[..., 0])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def so3_exp(phi):
    phi = np.asarray(phi, dtype=np.float64)
    th = np.linalg.norm(phi, axis=-1)[..., None, None]
    K = _hat(phi)
    small = th < 1e-8
    ths = np.where(small, 1.0, th)
    A = np.where(small, 1.0 - th * th / 6.0, np.sin(ths) / ths)
    B = np.where(small, 0.5 - th * th / 24.0, (1.0 - np.cos(ths)) / (ths * ths))
    return np.eye(3) + A * K + B * (K @ K)


def so3_right_jacobian(phi):
    th = np.linalg.norm(phi, axis=-1)[..., None, None]
    K = _hat(phi)
    small = th < 1e-8
    ths = np.where(small, 1.0, th)
    A = np.where(small, 0.5 - th * th / 24.0, (1.0 - np.cos(ths)) / (ths * ths))
    B = np.where(small, 1.0 / 6.0 - th * th / 120.0, (ths - np.sin(ths)) / (ths ** 3))
    return np.eye(3) - A * K + B * (K @ K)


def quat_xyzw_to_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def matrix_to_quat_xyzw(R):
    """Batch rotation matrices (..., 3, 3) -> unit quaternions (..., 4) in x,y,z,w order with w >= 0."""
    R = np.asarray(R, dtype=np.float64)
    out = np.empty(R.shape[:-2] + (4,))
    flat_R = R.reshape(-1, 3, 3)
    flat_o = out.reshape(-1, 4)
    for i, M in enumerate(flat_R):
        t = np.trace(M)
        if t > 0:
            s = np.sqrt(t + 1.0) * 2
            q = np.array([(M[2, 1] - M[1, 2]) / s, (M[0, 2] - M[2, 0]) / s, (M[1, 0] - M[0, 1]) / s, 0.25 * s])
        elif M[0, 0] > M[1, 1] and M[0, 0] > M[2, 2]:
            s = np.sqrt(1.0 + M[0, 0] - M[1, 1] - M[2, 2]) * 2
            q = np.array([0.25 * s, (M[0, 1] + M[1, 0]) / s, (M[0, 2] + M[2, 0]) / s, (M[2, 1] - M[1, 2]) / s])
        elif M[1, 1] > M[2, 2]:
            s = np.sqrt(1.0 + M[1, 1] - M[0, 0] - M[2, 2]) * 2
            q = np.array([(M[0, 1] + M[1, 0]) / s, 0.25 * s, (M[1, 2] + M[2, 1]) / s, (M[0, 2] - M[2, 0]) / s])
        else:
            s = np.sqrt(1.0 + M[2, 2] - M[0, 0] - M[1, 1]) * 2
            q = np.array([(M[0, 2] + M[2, 0]) / s, (M[1, 2] + M[2, 1]) / s, 0.25 * s, (M[1, 0] - M[0, 1]) / s])
        if q[3] < 0:
            q = -q
        flat_o[i] = q / np.linalg.norm(q)
    return out


class Trajectory:
    """Analytic IMU trajectory: R_wi(t) = R_base exp(phi(t)), p_wi(t) = p_base + s(t); sums of three sinusoids per axis."""

    def __init__(self, rng, R_base, p_base, rot_amp=0.15, pos_amp=0.10):
        self.R_base, self.p_base = R_base, p_base
        self.f_rot = rng.uniform(0.2, 1.5, size=(3, 3))
        self.f_pos = rng.uniform(0.2, 1.5, size=(3, 3))
        self.ph_rot = rng.uniform(0, 2 * np.pi, size=(3, 3))
        self.ph_pos = rng.uniform(0, 2 * np.pi, size=(3, 3))
        self.a_rot = rng.uniform(0.5, 1.0, size=(3, 3)) * rot_amp / 3.0
        self.a_pos = rng.uniform(0.5, 1.0, size=(3, 3)) * pos_amp / 3.0

    @staticmethod
    def _sin(t, a, f, ph, order):
        w = 2 * np.pi * f
        arg = w[None] * np.asarray(t)[..., None, None] + ph[None]
        if order == 0:
            v = a * np.sin(arg)
        elif order == 1:
            v = a * w * np.cos(arg)
        else:
            v = -a * w * w * np.sin(arg)
        return v.sum(-1)

    def phi(self, t, order=0):
        return self._sin(t, self.a_rot, self.f_rot, self.ph_rot, order)

    def R_wi(self, t):
        return self.R_base @ so3_exp(self.phi(t))

    def p_wi(self, t, order=0):
        s = self._sin(t, self.a_pos, self.f_pos, self.ph_pos, order)
        return s + self.p_base if order == 0 else s

    def omega_body(self, t):
        phi, dphi = self.phi(t), self.phi(t, 1)
        return (so3_right_jacobian(phi) @ dphi[..., None])[..., 0]


def make_dataset(cfg: SyntheticConfig) -> dict:
    rng = np.random.default_rng(cfg.seed)
    W, H = cfg.image_size
    ld_true = cfg.line_delay_truth if cfg.line_delay_truth is not None else 1.0 / cfg.fps / H
    # board: planar grid in z = 0, centred, ids row-major; homogeneous points
    cols, rows = cfg.grid
    gx, gy = np.meshgrid((np.arange(cols) - (cols - 1) / 2) * cfg.square_m, (np.arange(rows) - (rows - 1) / 2) * cfg.square_m)
    board = np.stack([gx.ravel(), gy.ravel(), np.zeros(cols * rows), np.ones(cols * rows)], -1)
    C = board.shape[0]
    # truth extrinsics: T_i_c (camera pose in the IMU frame), README dataset 1
    q_ic = np.array([-0.007, -0.708, 0.706, 0.005]); q_ic /= np.linalg.norm(q_ic)
    R_ic = quat_xyzw_to_matrix(q_ic)
    t_ic = np.array([0.007, -0.022, 0.001])
    # camera looks down on the board from ~0.5 m; IMU base pose follows from T_wc = T_wi * T_i_c
    R_wc_base = np.diag([1.0, -1.0, -1.0])
    p_wc_base = np.array([0.0, 0.0, 0.5])
    R_wi_base = R_wc_base @ R_ic.T
    p_wi_base = p_wc_base - R_wi_base @ t_ic
    traj = Trajectory(rng, R_wi_base, p_wi_base)
    gravity = np.array([0.0, 0.0, 9.81])

    frame_t = np.arange(cfg.n_frames) / cfg.fps
    # rolling shutter observation times in the reference's model: physical offset = y * ld * dt (dt_so3 == dt_r3 here)
    dt_phys = cfg.dt_so3_s
    uv = np.zeros((cfg.n_frames, C, 2))
    y_row = np.full((cfg.n_frames, C), H / 2.0)
    X = board[:, :3]
    for _ in range(4):
        t_obs = frame_t[:, None] + y_row * ld_true * dt_phys
        R = traj.R_wi(t_obs.ravel()).reshape(cfg.n_frames, C, 3, 3)
        p = traj.p_wi(t_obs.ravel()).reshape(cfg.n_frames, C, 3)
        q_imu = np.einsum("fcji,fcj->fci", R, X[None] - p)           # R_wi^T (X - p_wi)
        p_cam = np.einsum("ji,fcj->fci", R_ic, q_imu - t_ic)            # R_ic^T (q - t_ic)
        uv, valid = cm.project(cfg.model, cfg.intrinsics, p_cam)
        y_row = uv[..., 1]
    assert valid.all(), "synthetic trajectory left the camera model's valid domain"
    uv_noisy = uv + rng.normal(0.0, cfg.corner_noise_px, size=uv.shape)

    # per-frame pose priors (PnP-like): T_wc at the frame timestamp + noise
    R_wi_f = traj.R_wi(frame_t)
    p_wi_f = traj.p_wi(frame_t)
    R_wc = R_wi_f @ R_ic
    p_wc = p_wi_f + (R_wi_f @ t_ic)
    R_wc_n = R_wc @ so3_exp(rng.normal(0.0, cfg.pose_noise_rad, size=(cfg.n_frames, 3)))
    p_wc_n = p_wc + rng.normal(0.0, cfg.pose_noise_m, size=p_wc.shape)
    q_wc = matrix_to_quat_xyzw(R_wc_n)

    # IMU streams on the IMU clock; camera time = imu time + offset
    duration = frame_t[-1]
    n_imu = int(np.floor((duration + 0.5) * cfg.imu_rate_hz)) + 1
    t_cam_clock = np.arange(n_imu) / cfg.imu_rate_hz - 0.25
    R_i = traj.R_wi(t_cam_clock)
    acc = np.einsum("nji,nj->ni", R_i, traj.p_wi(t_cam_clock, 2) + gravity)
    gyr = traj.omega_body(t_cam_clock)
    b_a = np.array([0.05, -0.03, 0.02]); b_g = np.array([2e-3, -1e-3, 5e-4])
    sig_a = 1.5e-2 * np.sqrt(cfg.imu_rate_hz); sig_g = 1.1e-3 * np.sqrt(cfg.imu_rate_hz)
    if cfg.imu_noise:
        acc = acc + rng.normal(0.0, sig_a, size=acc.shape)
        gyr = gyr + rng.normal(0.0, sig_g, size=gyr.shape)
    acc = acc + b_a
    gyr = gyr + b_g
    imu_t = t_cam_clock - cfg.time_offset_imu_to_cam_s

    # initial T_i_c: rotation perturbed, translation zero (app :170, quirk q8)
    axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
    R_ic_init = R_ic @ so3_exp(axis * cfg.tic_rot_perturb_rad)
    q_ic_init = matrix_to_quat_xyzw(R_ic_init)
    T_ic_init = np.concatenate([q_ic_init, np.zeros(3)])

    offsets = (np.arange(cfg.n_frames + 1) * C).astype(np.int32)
    point_ids = np.tile(np.arange(C, dtype=np.int32), cfg.n_frames)
    return dict(
        name=cfg.name, config=cfg, model=cfg.model, intrinsics=np.asarray(cfg.intrinsics, dtype=np.float64), image_size=(W, H), fps=cfg.fps,
        board_xyzw=board, frame_t=frame_t, corner_offsets=offsets, point_ids=point_ids, uv=uv_noisy.reshape(-1, 2).copy(),
        q_wc=q_wc, p_wc=p_wc_n, imu_t=imu_t, accel=acc, gyro=gyr,
        dt_so3_s=cfg.dt_so3_s, dt_r3_s=cfg.dt_r3_s, std_so3=sig_g if cfg.imu_noise else 1.0, std_r3=sig_a if cfg.imu_noise else 1.0,
        time_offset_imu_to_cam_s=cfg.time_offset_imu_to_cam_s, init_line_delay_s=ld_true * cfg.line_delay_init_scale,
        T_i_c_init=T_ic_init, acc_bias=b_a, gyr_bias=b_g, gravity=gravity,
        truth=dict(T_i_c=np.concatenate([q_ic, t_ic]), line_delay=ld_true, gravity=gravity),
    )


# ---- static multi-pose IMU sequence (input of static_imu_calibration) -----------------------------------------------------------
# A still initial period, then static poses joined by minimum-jerk pure rotations about a fixed body axis: the specific force is
# R^T g (no lever arm) and the body rate is s'(tau) phi.  Raw readings invert the calibration model of the reference
# (calibrated = T K (raw - b), utils/types.h:170-323): raw = (T K)^-1 truth + b, plus seeded white noise (without noise the
# initial-interval variance is 0 and nothing would count as static).
STATIC_IMU_TRUTH = dict(
    acc=np.array([1.5e-3, -2.0e-3, 1.0e-3, 1.004, 0.997, 1.006, 0.06, -0.09, 0.12]),                 # misYZ, misZY, misZX, sX, sY, sZ, b
    gyr=np.array([2.0e-3, -1.0e-3, 1.5e-3, -2.5e-3, 1.0e-3, 3.0e-3, 0.995, 1.008, 1.003]),           # misYZ..misYX, sX, sY, sZ
    gyr_bias=np.array([0.004, -0.006, 0.003]))


def _triad_matrix(p, full):
    """ms = T K of ThreeAxisSensorCalibParams (types.h:225-246): T = [[1,-yz,zy],[xz,1,-zx],[-xy,yx,1]], K = diag(s)."""
    yz, zy, zx = p[0], p[1], p[2]
    xz, xy, yx = (p[3], p[4], p[5]) if full else (0.0, 0.0, 0.0)
    s = p[6:9] if full else p[3:6]
    T = np.array([[1.0, -yz, zy], [xz, 1.0, -zx], [-xy, yx, 1.0]])
    return T @ np.diag(s)


def make_static_imu_sequence(rate_hz=200.0, seed=7, n_poses=36, init_s=15.0, pose_s=(2.0, 4.0), move_s=(1.2, 2.0),
                             g_mag=9.81, acc_sigma=0.02, gyr_sigma=0.002) -> dict:
    """-> dict(t_s, accel (n,3), gyro (n,3), truth, g_mag, init_s, n_poses).  Deterministic for a given seed."""
    rng = np.random.default_rng(seed)
    dt = 1.0 / rate_hz
    g_w = np.array([0.0, 0.0, g_mag])
    R = np.eye(3)
    Rs, ws = [], []

    def hold(R, dur):
        k = int(round(dur * rate_hz))
        Rs.extend([R] * k); ws.extend([np.zeros(3)] * k)

    hold(R, init_s)
    for _ in range(n_poses):
        axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
        phi = axis * rng.uniform(0.6, 2.6)
        T = rng.uniform(*move_s)
        k = int(round(T * rate_hz))
        tau = (np.arange(k) + 0.5) / k
        s = 10 * tau ** 3 - 15 * tau ** 4 + 6 * tau ** 5
        sd = (30 * tau ** 2 - 60 * tau ** 3 + 30 * tau ** 4) / T
        Rs.extend(R @ so3_exp(s[:, None] * phi)); ws.extend(sd[:, None] * phi)
        R = R @ so3_exp(phi)
        hold(R, rng.uniform(*pose_s))
    Rs = np.array(Rs); ws = np.array(ws)
    n = len(Rs)
    t = np.arange(n) * dt
    f_true = np.einsum("nji,j->ni", Rs, g_w)                      # R^T g
    tr = STATIC_IMU_TRUTH
    Ma, Mg = _triad_matrix(tr["acc"], False), _triad_matrix(tr["gyr"], True)
    acc = f_true @ np.linalg.inv(Ma).T + tr["acc"][6:9] + rng.normal(scale=acc_sigma, size=(n, 3))
    gyr = ws @ np.linalg.inv(Mg).T + tr["gyr_bias"] + rng.normal(scale=gyr_sigma, size=(n, 3))
    return dict(t_s=t, accel=acc, gyro=gyr, truth=tr, g_mag=g_mag, init_s=init_s, n_poses=n_poses)


def static_imu_full_size(seed=11) -> dict:
    """1 kHz, about ten minutes: 30 s still, 40 poses of 2-4 s joined by 8-12 s rotations."""
    return make_static_imu_sequence(rate_hz=1000.0, seed=seed, n_poses=40, init_s=30.0, pose_s=(2.0, 4.0), move_s=(8.0, 12.0))


# ---- static IMU noise log (input of fit_allan_variance) --------------------------------------------------------------------------
ALLAN_TRUTH = dict(acc_white=2.0e-3, acc_walk=4.0e-5, acc_bias=(0.05, -0.08, 9.81), gyr_white=1.5e-4, gyr_walk=2.0e-6, gyr_bias=(3e-3, -2e-3, 1e-3))


def make_allan_log(rate_hz=200.0, duration_s=1200.0, seed=5, truth=ALLAN_TRUTH) -> dict:
    """A static IMU log: per axis, white noise of density `*_white` (units/sqrt(Hz)), a bias random walk of strength `*_walk`
    (units/s/sqrt(Hz)) and a constant bias.  In Allan terms the white noise gives sigma^2 = white^2 / tau (N = white) and the walk
    sigma^2 = walk^2 tau / 3 (K = walk / sqrt(3)).  Accelerometer in m/s^2, gyroscope in rad/s."""
    rng = np.random.default_rng(seed)
    n = int(round(duration_s * rate_hz)); dt = 1.0 / rate_hz
    t = np.arange(n) * dt
    out = {"t_s": t, "rate_hz": rate_hz, "truth": dict(truth)}
    for key in ("acc", "gyr"):
        white = truth[key + "_white"] * np.sqrt(rate_hz) * rng.standard_normal((n, 3))
        walk = np.cumsum(truth[key + "_walk"] * np.sqrt(dt) * rng.standard_normal((n, 3)), axis=0)
        out["accel" if key == "acc" else "gyro"] = np.asarray(truth[key + "_bias"]) + walk + white
    return out


def allan_small(seed=5) -> dict:
    """20 minutes at 200 Hz (240 000 samples)."""
    return make_allan_log(200.0, 1200.0, seed)


def allan_full_size(seed=6) -> dict:
    """2 hours at 400 Hz (2.88 M samples)."""
    return make_allan_log(400.0, 7200.0, seed)


# ---- radon checkerboard renderer ------------------------------------------------------------------------------------
# The board of the reference's resource/checkerboard_radon.png: (W + 1) x (H + 1) squares around W x H inner corners (14 x 9
# for the printed board), the top-left square white, black squares on the border rounded outward by a half disk, and three
# circle markers of diameter 0.36 squares near the centre.  In the board frame corner (i, j) sits at (i s, j s, 0) like the
# reference's scene points: x runs up the printed sheet (i = 0 is the bottom inner row), y runs right, z points into the sheet.
RADON_MARKER_RADIUS = 0.18   # squares


def radon_marker_cell(corners_x: int, corners_y: int):
    """Board cell (i, j) (corners (i..i+1, j..j+1)) of the L-shaped marker triple's vertex: a black circle in a white square.
    The arms are the cells (i + 1, j) and (i, j + 1), white circles in black squares."""
    return corners_y // 2 - 1, corners_x // 2 - 1


def radon_board_points(corners_x: int, corners_y: int, square_m: float):
    """(H W, 3) board points in id order id = i W + j."""
    i, j = np.meshgrid(np.arange(corners_y), np.arange(corners_x), indexing="ij")
    return np.stack([i.ravel() * square_m, j.ravel() * square_m, np.zeros(i.size)], -1)


def radon_board_shade(xb, yb, corners_x: int, corners_y: int, square_m: float, markers: bool = True, marker_cell=None):
    """Reflectance in [0, 1] (0 black) at board-frame points (xb, yb).  `marker_cell` moves the marker triple's vertex to another
    cell (a board that is not the radon board)."""
    W, H = corners_x, corners_y
    u = yb / square_m + 1.0                     # printed columns from the left edge, 0 .. W + 1
    v = (H - 1) - xb / square_m + 1.0           # printed rows from the top edge, 0 .. H + 1
    C, R = np.floor(u), np.floor(v)
    inside = (C >= 0) & (C <= W) & (R >= 0) & (R <= H)
    black = ((R + C) % 2 == 1) & inside
    du, dv = u - C - 0.5, v - R - 0.5           # offset from the square's centre, squares
    outward = ((C == 0) & (du < 0)) | ((C == W) & (du > 0)) | ((R == 0) & (dv < 0)) | ((R == H) & (dv > 0))
    black &= ~outward | (du * du + dv * dv <= 0.25)
    if markers:
        mi, mj = radon_marker_cell(W, H) if marker_cell is None else marker_cell
        dot = du * du + dv * dv <= RADON_MARKER_RADIUS ** 2
        for ci, cj in ((mi, mj), (mi + 1, mj), (mi, mj + 1)):
            black ^= dot & (C == cj + 1) & (R == H - 1 - ci)
    return np.where(black, 0.0, 1.0)


def unproject_grid(model: int, intr, uv, iters: int = 30):
    """Camera-frame rays (x, y, 1) of pixels uv (..., 2) by damped Newton on cm.project with a central-difference Jacobian."""
    uv = np.asarray(uv, dtype=np.float64)
    k = np.asarray(intr, dtype=np.float64)
    f = k[0]
    cx, cy = (k[2], k[3]) if model in (cm.FOV, cm.DIVISION_UNDISTORTION) else (k[3], k[4])
    x = np.stack([(uv[..., 0] - cx) / f, (uv[..., 1] - cy) / f], -1)
    one = np.ones(uv.shape[:-1])

    def proj(xy):
        return cm.project(model, k, np.stack([xy[..., 0], xy[..., 1], one], -1))[0]
    h = 1e-6
    for _ in range(iters):
        r = proj(x) - uv
        J = np.stack([(proj(x + [h, 0]) - proj(x - [h, 0])) / (2 * h), (proj(x + [0, h]) - proj(x - [0, h])) / (2 * h)], -1)
        det = J[..., 0, 0] * J[..., 1, 1] - J[..., 0, 1] * J[..., 1, 0]
        dx = (J[..., 1, 1] * r[..., 0] - J[..., 0, 1] * r[..., 1]) / det
        dy = (-J[..., 1, 0] * r[..., 0] + J[..., 0, 0] * r[..., 1]) / det
        step = np.stack([dx, dy], -1)
        n = np.linalg.norm(step, axis=-1, keepdims=True)
        x = x - step * np.minimum(1.0, 0.5 / np.maximum(n, 1e-300))   # damped: at most 0.5 in normalised units per step
        if np.nanmax(np.abs(r)) < 1e-9:
            break
    ok = np.linalg.norm(proj(x) - uv, axis=-1) < 1e-6
    return np.stack([x[..., 0], x[..., 1], one], -1), ok


def radon_view_pose(corners_x: int, corners_y: int, square_m: float, distance_m: float, tilt_deg: float = 0.0, tilt_axis_deg: float = 0.0,
                    roll_deg: float = 0.0, offset_m=(0.0, 0.0)):
    """(R_cb, t_cb) of a camera `distance_m` in front of the board centre: the printed sheet upright in the image at roll 0, tilted
    by `tilt_deg` about an in-plane axis at `tilt_axis_deg`, rolled about the optical axis, and the board shifted by `offset_m`."""
    R_bc0 = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])   # camera x = board y, camera y = -board x, camera z = board z
    a = np.deg2rad(tilt_axis_deg)
    tilt = so3_exp(np.deg2rad(tilt_deg) * np.array([np.cos(a), np.sin(a), 0.0]))
    roll = so3_exp(np.array([0.0, 0.0, np.deg2rad(roll_deg)]))
    R_cb = roll @ tilt @ R_bc0.T
    centre = np.array([(corners_y - 1) * square_m / 2, (corners_x - 1) * square_m / 2, 0.0])
    t_cb = np.array([offset_m[0], offset_m[1], distance_m]) - R_cb @ centre
    return R_cb, t_cb


def render_radon_board(model: int, intr, size, R_cb, t_cb, corners_x: int = 14, corners_y: int = 9, square_m: float = 0.03,
                       supersample: int = 4, blur_sigma_px: float = 0.0, noise_sigma_dn: float = 0.0, seed: int = 0, markers: bool = True,
                       black_dn: float = 30.0, white_dn: float = 220.0, rays=None, marker_cell=None):
    """uint8 (height, width) image of the radon board seen by the camera (model, intr) at board-to-camera pose (R_cb, t_cb), by
    supersampled ray casting (supersample^2 stratified, jittered rays per pixel, pixel centres at integer coordinates); optional
    Gaussian blur and noise.  Returns (image, truth uv (H W, 2) in id order, truth valid).  `rays` reuses camera_rays(...) of the same camera."""
    width, height = size
    if rays is None:
        rays = camera_rays(model, intr, size, supersample)
    d, ok = rays
    R_cb, t_cb = np.asarray(R_cb, float), np.asarray(t_cb, float)
    n = R_cb[:, 2]
    lam = (n @ t_cb) / (d @ n)
    pb = (lam[..., None] * d - t_cb) @ R_cb                       # R_cb^T (lam d - t)
    hit = ok & (lam > 0)
    shade = np.where(hit, radon_board_shade(pb[..., 0], pb[..., 1], corners_x, corners_y, square_m, markers, marker_cell), 1.0)
    img = shade.reshape(height, supersample, width, supersample).mean(axis=(1, 3))
    img = black_dn + (white_dn - black_dn) * img
    if blur_sigma_px > 0:
        from scipy.ndimage import gaussian_filter
        img = gaussian_filter(img, blur_sigma_px, mode="nearest")
    if noise_sigma_dn > 0:
        img = img + np.random.default_rng(seed).normal(0.0, noise_sigma_dn, img.shape)
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    pc = radon_board_points(corners_x, corners_y, square_m) @ R_cb.T + t_cb
    uv, valid = cm.project(model, intr, pc)
    valid = valid & (pc[:, 2] > 0) & (uv[:, 0] >= 0) & (uv[:, 0] <= width - 1) & (uv[:, 1] >= 0) & (uv[:, 1] <= height - 1)
    return img, uv, valid


_RAYS = {}


def camera_rays(model: int, intr, size, supersample: int = 4):
    """Rays of the supersampled pixel grid (height * ss, width * ss, 3) and their validity, cached per camera.  Each pixel's ss x ss
    cells get one ray at a uniformly random point inside the cell (a fixed seed): a regular grid would put every edge of an
    axis-aligned square at the same sub-cell phase and bias its rendered position by up to 1 / (2 ss) px."""
    key = (model, tuple(float(x) for x in intr), tuple(size), supersample)
    if key not in _RAYS:
        width, height = size
        cells = np.arange(supersample) / supersample - 0.5
        jit = np.random.default_rng(12345).uniform(0.0, 1.0 / supersample, (2, height * supersample, width * supersample))
        uu = (np.arange(width)[:, None] + cells[None]).ravel()[None, :] + jit[0]
        vv = (np.arange(height)[:, None] + cells[None]).ravel()[:, None] + jit[1]
        _RAYS.clear()
        _RAYS[key] = unproject_grid(model, intr, np.stack([uu, vv], -1))
    return _RAYS[key]


# ---- Kalibr AprilGrid (BoardType::APRILTAG) ------------------------------------------------------------------------------------------
# tags_x x tags_y tag36h11 tags of side s, spacing 0.3 s: tag t = tags_x y + x has its lower-left corner at (1.3 s x, 1.3 s y) in the
# board frame (x right, y up the printed sheet, z out of it), and a black square of side 0.3 s fills every gap crossing, the outer
# ones included (Kalibr's corner squares, which make every tag corner an X-junction).
def tag36h11_codes():
    """The 587 codes of csrc/icc_tag36h11.h (the codebook the GPU decoder uses)."""
    import re
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "icc_tag36h11.h")
    return np.array([int(x, 16) for x in re.findall(r"0x([0-9a-f]+)ull", open(path).read())], dtype=np.uint64)


def aprilgrid_board_points(tags_x: int, tags_y: int, tag_m: float):
    """(4 tags_x tags_y, 3) board points in point-id order (t << 2) + i, i = bottom-left, bottom-right, top-right, top-left."""
    i = np.arange(4 * tags_x * tags_y)
    t, c = i >> 2, i & 3
    x = (t % tags_x) * tag_m * 1.3 + np.array([0.0, tag_m, tag_m, 0.0])[c]
    y = (t // tags_x) * tag_m * 1.3 + np.array([0.0, 0.0, tag_m, tag_m])[c]
    return np.stack([x, y, np.zeros_like(x)], -1)


def aprilgrid_shade(xb, yb, tags_x: int, tags_y: int, tag_m: float, tag_ids=None, codes=None):
    """Reflectance in [0, 1] (0 black) at board-frame points.  tag_ids[t] is the id drawn at position t (default t).  A code's first
    (most significant) bit is the top-left data cell with the board's y up; 1 is white."""
    codes = tag36h11_codes() if codes is None else codes
    ids = np.arange(tags_x * tags_y) if tag_ids is None else np.asarray(tag_ids)
    pitch = 1.3 * tag_m
    tx, ty = np.floor(xb / pitch), np.floor(yb / pitch)
    fx, fy = (xb - tx * pitch) / tag_m, (yb - ty * pitch) / tag_m
    in_x, in_y = (tx >= 0) & (tx < tags_x), (ty >= 0) & (ty < tags_y)
    tag = in_x & in_y & (fx < 1) & (fy < 1)
    crossing = (tx >= -1) & (tx < tags_x) & (ty >= -1) & (ty < tags_y) & (fx >= 1) & (fy >= 1)
    cx = np.clip(np.floor(fx * 10), 0, 9).astype(np.int64)
    cy = 9 - np.clip(np.floor(fy * 10), 0, 9).astype(np.int64)          # cell row from the tag's top
    data = tag & (cx >= 2) & (cx <= 7) & (cy >= 2) & (cy <= 7)
    t = (np.clip(ty, 0, tags_y - 1) * tags_x + np.clip(tx, 0, tags_x - 1)).astype(np.int64)
    code = codes[ids[t]]
    k = ((cy - 2) * 6 + (cx - 2)).clip(0, 35)
    bit = (code >> (35 - k).astype(np.uint64)) & np.uint64(1)
    white = ~(tag | crossing) | (data & (bit == 1))
    return np.where(white, 1.0, 0.0)


def aprilgrid_view_pose(tags_x: int, tags_y: int, tag_m: float, distance_m: float, tilt_deg: float = 0.0, tilt_axis_deg: float = 0.0,
                        roll_deg: float = 0.0, offset_m=(0.0, 0.0)):
    """(R_cb, t_cb) of a camera `distance_m` in front of the grid's centre: the sheet upright (board y up the image) at roll 0,
    tilted by `tilt_deg` about an in-plane axis at `tilt_axis_deg`, rolled about the optical axis, and the board shifted by `offset_m`."""
    a = np.deg2rad(tilt_axis_deg)
    tilt = so3_exp(np.deg2rad(tilt_deg) * np.array([np.cos(a), np.sin(a), 0.0]))
    roll = so3_exp(np.array([0.0, 0.0, np.deg2rad(roll_deg)]))
    R_cb = roll @ tilt @ np.diag([1.0, -1.0, -1.0])
    centre = np.array([(tags_x * 1.3 - 0.3) * tag_m / 2, (tags_y * 1.3 - 0.3) * tag_m / 2, 0.0])
    t_cb = np.array([offset_m[0], offset_m[1], distance_m]) - R_cb @ centre
    return R_cb, t_cb


def render_aprilgrid(model: int, intr, size, R_cb, t_cb, tags_x: int = 6, tags_y: int = 6, tag_m: float = 0.04, supersample: int = 4,
                     blur_sigma_px: float = 0.0, noise_sigma_dn: float = 0.0, seed: int = 0, black_dn: float = 30.0, white_dn: float = 220.0,
                     tag_ids=None, rays=None):
    """uint8 (height, width) image of the AprilGrid seen by the camera (model, intr) at board-to-camera pose (R_cb, t_cb), by the
    supersampled ray casting of render_radon_board; optional Gaussian blur and noise.  Returns (image, truth uv (4 tags_x tags_y, 2)
    in point-id order, truth valid)."""
    width, height = size
    if rays is None:
        rays = camera_rays(model, intr, size, supersample)
    d, ok = rays
    R_cb, t_cb = np.asarray(R_cb, float), np.asarray(t_cb, float)
    n = R_cb[:, 2]
    lam = (n @ t_cb) / (d @ n)
    pb = (lam[..., None] * d - t_cb) @ R_cb
    hit = ok & (lam > 0)
    shade = np.where(hit, aprilgrid_shade(pb[..., 0], pb[..., 1], tags_x, tags_y, tag_m, tag_ids), 1.0)
    img = shade.reshape(height, supersample, width, supersample).mean(axis=(1, 3))
    img = black_dn + (white_dn - black_dn) * img
    if blur_sigma_px > 0:
        from scipy.ndimage import gaussian_filter
        img = gaussian_filter(img, blur_sigma_px, mode="nearest")
    if noise_sigma_dn > 0:
        img = img + np.random.default_rng(seed).normal(0.0, noise_sigma_dn, img.shape)
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    pc = aprilgrid_board_points(tags_x, tags_y, tag_m) @ R_cb.T + t_cb
    uv, valid = cm.project(model, intr, pc)
    valid = valid & (pc[:, 2] > 0) & (uv[:, 0] >= 0) & (uv[:, 0] <= width - 1) & (uv[:, 1] >= 0) & (uv[:, 1] <= height - 1)
    return img, uv, valid
