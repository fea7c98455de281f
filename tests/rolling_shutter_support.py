"""Test infrastructure of the pose step's rolling shutter (icc_set_pose_rolling_shutter).

- `host_math_lib()`: the product's rolling-shutter header (csrc/icc_rolling_shutter_math.cuh) compiled for the CPU, built once per process
  into a temporary directory.
- `rs_sequence()`: a synthetic sequence with a physical rolling shutter: a smooth handheld-like trajectory over a planar board, every corner
  projected with the pose at its own row time (solved by fixed-point iteration), so the constant-velocity model of the product is only an
  approximation of it.
- `RsPoseOracle`: the oracle of icc_estimate_board_poses / icc_optimize_board_points with a rolling shutter, with the method shapes of
  `_capi.CApi`.  The global-shutter pass is `wide_angle_support.PoseOracle` (the C++ oracle, or NumPy for the tangent residual); the
  neighbour velocities, the rolling-shutter passes and the board-point refinement are restated here in NumPy, with rotation matrices,
  a left-increment Levenberg-Marquardt and scipy's rotation log.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial.transform import Rotation

from openimucameracalibrator_b200 import camera_models as cm
from wide_angle_support import HUBER, PoseOracle, _exp, oracle_basis, oracle_bearings

HERE = os.path.dirname(os.path.abspath(__file__))
W, H, FPS = 960, 540, 60.0
LINE_DELAY = 1.0 / FPS / H                       # 30.9 us per row: one readout per frame interval
_LIB = None


def host_math_lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_rolling_shutter_"), "librs_host_math.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "rolling_shutter", "rs_host_math.cu")])
        _LIB = ctypes.CDLL(out)
    return _LIB


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def _c(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def product_rs_residual(tangent, meas, q_xyzw, X, t, wu, tau):
    """-> (r[2], front, J[2,6]) of the product header (right increment)."""
    a = [_c(v) for v in (meas, q_xyzw, X, t, wu)]
    r = np.zeros(2); J = np.zeros(12)
    lib = host_math_lib(); lib.rs_residual.restype = ctypes.c_int
    front = lib.rs_residual(int(tangent), *[_dp(v) for v in a], ctypes.c_double(tau), _dp(r), _dp(J))
    return r, bool(front), J.reshape(2, 6)


def product_rs_transform(P0, wu, tau):
    P = np.zeros(3)
    host_math_lib().rs_transform(_dp(_c(P0)), _dp(_c(wu)), ctypes.c_double(tau), _dp(P))
    return P


def product_rs_velocity(qa, pa, ta, qb, pb, tb, qf):
    wu = np.zeros(6)
    host_math_lib().rs_velocity(_dp(_c(qa)), _dp(_c(pa)), ctypes.c_double(ta), _dp(_c(qb)), _dp(_c(pb)), ctypes.c_double(tb), _dp(_c(qf)), _dp(wu))
    return wu


# ---- the synthetic rolling-shutter sequence ------------------------------------------------------------------------------------------
def board(cols=9, rows=7, sq=0.021):
    gx, gy = np.meshgrid((np.arange(cols) - (cols - 1) / 2) * sq, (np.arange(rows) - (rows - 1) / 2) * sq)
    return np.stack([gx.ravel(), gy.ravel(), np.zeros(cols * rows), np.ones(cols * rows)], -1)


class Trajectory:
    """Camera over the board z = 0, looking down: R_wc(t) = R0 exp(theta(t)), p_wc(t) = p0 + d(t), sums of sinusoids.
    rot_amp (rad) and pos_amp (m) set the motion; 0 is a motionless camera."""

    def __init__(self, seed=0, rot_amp=0.1, pos_amp=0.03, height=0.42, freqs=(2.0, 3.5)):
        rng = np.random.default_rng(seed)
        self.R0 = Rotation.from_rotvec([np.pi, 0.0, 0.0]).as_matrix()
        self.p0 = np.array([0.0, 0.0, height])
        m = 1 if len(freqs) == 2 else len(freqs)            # (lo, hi): one random frequency per axis; a longer tuple: all of them on every axis
        f = rng.uniform(*freqs, (3, 1)) if len(freqs) == 2 else np.tile(np.asarray(freqs, dtype=np.float64), (3, 1))
        self.fr = f; self.phr = rng.uniform(0, 2 * np.pi, (3, m)); self.ar = rot_amp * rng.uniform(0.7, 1.0, (3, m))
        self.fp = 0.75 * f; self.php = rng.uniform(0, 2 * np.pi, (3, m)); self.ap = pos_amp * rng.uniform(0.7, 1.0, (3, m)) * np.array([[1], [1], [0.5]])

    def R(self, t):
        return self.R0 @ _exp((self.ar * np.sin(2 * np.pi * self.fr * t + self.phr)).sum(1))

    def p(self, t):
        return self.p0 + (self.ap * np.sin(2 * np.pi * self.fp * t + self.php)).sum(1)

    def velocity(self, t, h=1e-5):
        """camera-frame (w, u) at t (central differences of the closed-form trajectory, ~1e-9 accurate)"""
        R, Rm = self.R(t), self.R(t - h)
        w = R.T @ Rm @ Rotation.from_matrix(Rm.T @ self.R(t + h)).as_rotvec() / (2 * h)
        u = R.T @ (self.p(t + h) - self.p(t - h)) / (2 * h)
        return w, u


def _project_rs(model, k, traj, t, X, line_delay):
    """Pixels of board points X seen by a rolling shutter at frame time t: row v is exposed at t + v line_delay (fixed point in v)."""
    tau = np.zeros(len(X))
    for _ in range(8):
        pc = np.stack([traj.R(t + tt).T @ (x - traj.p(t + tt)) for x, tt in zip(X, tau)])
        px, valid = cm.project(model, k, pc)
        tau = px[:, 1] * line_delay
    return px, valid


def rs_sequence(model, k, n_frames=60, seed=0, noise_px=0.2, line_delay=LINE_DELAY, rot_amp=0.1, pos_amp=0.03, t0=1.0, freqs=(2.0, 3.5)):
    """60 fps views of the board; returns dict(board, off, ids, uv, frame_t, q_wc, p_wc, w, u (truth at each frame time), mean_row)."""
    rng = np.random.default_rng(seed + 1000)
    traj = Trajectory(seed, rot_amp, pos_amp, freqs=freqs)
    B = board(); X = B[:, :3]; C = len(X)
    t = t0 + np.arange(n_frames) / FPS
    uv, q, p, w, u = [], [], [], [], []
    for tf in t:
        px, valid = _project_rs(model, k, traj, tf, X, line_delay)
        assert valid.all() and (px > 0).all() and (px[:, 0] < W).all() and (px[:, 1] < H).all(), "the board leaves the image"
        uv.append(px + rng.normal(0, noise_px, px.shape))
        R = traj.R(tf)
        q.append(Rotation.from_matrix(R).as_quat()); p.append(traj.p(tf))
        wi, ui = traj.velocity(tf); w.append(wi); u.append(ui)
    uv = np.concatenate(uv)
    return dict(board=B, off=(np.arange(n_frames + 1) * C).astype(np.int32), ids=np.tile(np.arange(C, dtype=np.int32), n_frames), uv=uv,
                frame_t=t, q_wc=np.array(q), p_wc=np.array(p), w=np.array(w), u=np.array(u), mean_row=float(uv[:, 1].mean()), traj=traj)


# ---- the oracle --------------------------------------------------------------------------------------------------------------------
def _R(q):
    return Rotation.from_quat(q).as_matrix()


def view_velocities(frame_t, q_wc, p_wc, valid):
    """The neighbour rule of icc_set_pose_rolling_shutter -> (vel[n,6], nbr[n]: neighbours used, -1 for an invalid view)."""
    t = np.asarray(frame_t, dtype=np.float64); n = t.size
    order = np.argsort(t, kind="stable"); ts = t[order]
    gaps = np.diff(ts); gaps = gaps[gaps > 0]
    max_gap = 2.5 * np.median(gaps) if gaps.size else -1.0
    vel = np.zeros((n, 6)); nbr = np.full(n, -1)
    for i, f in enumerate(order):
        if not valid[f]:
            continue
        a = b = None
        for j in range(i - 1, -1, -1):
            if ts[i] - ts[j] > max_gap:
                break
            if ts[i] - ts[j] > 0 and valid[order[j]]:
                a = j; break
        for j in range(i + 1, n):
            if ts[j] - ts[i] > max_gap:
                break
            if ts[j] - ts[i] > 0 and valid[order[j]]:
                b = j; break
        nbr[f] = (a is not None) + (b is not None)
        if nbr[f] == 0:
            continue
        fa, ta = (order[a], ts[a]) if a is not None else (f, ts[i])
        fb, tb = (order[b], ts[b]) if b is not None else (f, ts[i])
        Ra, Rb, Rf = _R(q_wc[fa]), _R(q_wc[fb]), _R(q_wc[f])
        vel[f, :3] = Rf.T @ Ra @ Rotation.from_matrix(Ra.T @ Rb).as_rotvec() / (tb - ta)
        vel[f, 3:] = Rf.T @ (p_wc[fb] - p_wc[fa]) / (tb - ta)
    return vel, nbr


def _rs_points(R, t, X, tau, w, u):
    """P(tau) = exp(-tau [w]x)(R X + t - tau u) for every corner, and the A(tau) matrices"""
    A = Rotation.from_rotvec(-tau[:, None] * w[None]).as_matrix()
    return np.einsum("nij,nj->ni", A, X @ R.T + t - tau[:, None] * u[None]), A


def _errors(P, meas, tangent):
    """residuals r[n,2], front[n] and rows a0, a1 [n,3] of d r / d P"""
    if tangent:
        e1, e2 = oracle_basis(meas)
        s = np.einsum("ij,ij->i", meas, P)
        r = np.stack([np.einsum("ij,ij->i", e1, P), np.einsum("ij,ij->i", e2, P)], -1) / s[:, None]
        return r, s > 0, (e1 - r[:, :1] * meas) / s[:, None], (e2 - r[:, 1:] * meas) / s[:, None]
    iz = 1.0 / P[:, 2]; x, y = P[:, 0] * iz, P[:, 1] * iz
    r = np.stack([x - meas[:, 0], y - meas[:, 1]], -1)
    z = np.zeros_like(iz)
    return r, P[:, 2] > 0, np.stack([iz, z, -x * iz], -1), np.stack([z, iz, -y * iz], -1)


def _cost(r, front):
    rn = np.linalg.norm(r, axis=1)
    return float(np.sum(np.where(rn <= HUBER, 0.5 * rn * rn, HUBER * rn - 0.5 * HUBER * HUBER)) + 1e6 * np.sum(~front))


def _lm(x, res_jac, apply, iters=200):
    """Levenberg-Marquardt on the Huber(1.345) cost to a 1e-16 relative stall; res_jac(x) -> (r, front, J[n,2,k])"""
    r, fr, J = res_jac(x); cost = _cost(r, fr); lam = 1e-3
    for _ in range(iters):
        rn = np.linalg.norm(r, axis=1); wt = np.where(rn <= HUBER, 1.0, HUBER / np.maximum(rn, 1e-300))
        Jw = J[fr] * np.sqrt(wt[fr])[:, None, None]; rw = r[fr] * np.sqrt(wt[fr])[:, None]
        Hm = np.einsum("nij,nik->jk", Jw, Jw); g = np.einsum("nij,ni->j", Jw, rw)
        stepped = False
        while lam < 1e16:
            dx = np.linalg.solve(Hm + lam * np.diag(np.diag(Hm) + 1e-12), -g)
            xn = apply(x, dx); rn2, frn, Jn = res_jac(xn); cn = _cost(rn2, frn)
            if cn < cost:
                dec = cost - cn; x, r, fr, J, cost = xn, rn2, frn, Jn, cn; lam = max(lam * 0.1, 1e-14); stepped = True
                break
            lam *= 10
        if not stepped or dec <= 1e-16 * cost or dx @ dx < 1e-32:
            break
    return x


def refine_pose_rs(R, t, X, meas, tau, w, u, tangent):
    """the rolling-shutter pose refinement of one view: left increment R <- exp(d) R, t <- t + dt"""
    def res_jac(x):
        Rx, tx = x
        P, A = _rs_points(Rx, tx, X, tau, w, u)
        r, fr, a0, a1 = _errors(P, meas, tangent)
        a0 = np.einsum("nji,nj->ni", A, a0); a1 = np.einsum("nji,nj->ni", A, a1)        # A^T a
        RX = X @ Rx.T
        J = np.stack([np.concatenate([np.cross(RX, a0), a0], 1), np.concatenate([np.cross(RX, a1), a1], 1)], 1)
        return r, fr, J
    R, t = _lm((R, t), res_jac, lambda x, d: (_exp(d[:3]) @ x[0], x[1] + d[3:]))
    U, _, Vt = np.linalg.svd(R)
    return U @ Vt, t


def refine_point_rs(X, meas, Rs, cs, tau, w, u, tangent):
    """one board point with constant cameras (R_cw, centre c, velocities w, u per observation)"""
    def res_jac(Xp):
        A = Rotation.from_rotvec(-tau[:, None] * w).as_matrix()
        P = np.einsum("nij,nj->ni", A, np.einsum("nij,nj->ni", Rs, Xp - cs) - tau[:, None] * u)
        r, fr, a0, a1 = _errors(P, meas, tangent)
        M = np.einsum("nij,njk->nik", A, Rs)
        return r, fr, np.stack([np.einsum("ni,nij->nj", a0, M), np.einsum("ni,nij->nj", a1, M)], 1)
    return _lm(X, res_jac, lambda x, d: x + d)


class RsPoseOracle(PoseOracle):
    """PoseOracle with icc_set_pose_rolling_shutter, icc_get_pose_velocities and the rolling-shutter passes."""

    def __init__(self):
        super().__init__()
        self.line_delay = 0.0; self.frame_t = None; self.vel = None; self.n_static = 0; self._rs_board = None

    def set_pose_rolling_shutter(self, line_delay_s, frame_t_s=None):
        if not np.isfinite(line_delay_s) or line_delay_s < 0:
            raise ValueError("line delay")
        if line_delay_s == 0:
            self.line_delay, self.frame_t = 0.0, None
            return
        t = np.asarray(frame_t_s, dtype=np.float64).ravel()
        if t.size == 0 or not np.isfinite(t).all() or (t < 0).any():
            raise ValueError("frame times")
        self.line_delay, self.frame_t = float(line_delay_s), t

    def pose_velocities(self, n_frames):
        assert self.vel is not None and self.vel.shape[0] == n_frames
        return self.vel[:, :3].copy(), self.vel[:, 3:].copy(), self.n_static

    def get_board_points(self):
        return self._rs_board.copy() if self._rs_board is not None else super().get_board_points()

    def _meas(self, uv):
        if self.mode == 1:
            return oracle_bearings(self.model, self.k, uv)
        return self.cpp.pixels_to_normalized(uv)

    def _check(self, off):
        if self.line_delay > 0 and len(off) - 1 != self.frame_t.size:
            raise ValueError("n_frames differs from the view times")

    def _rs_pass(self, off, ids, uv, board, rules, q, p, e, v):
        """velocities from (q, p, v), then the refinement-only pass of every valid view -> (q, p, e, v, use, vel, nbr)"""
        mp, thresh, max_px = rules
        meas, ok = self._meas(uv)
        vel, nbr = view_velocities(self.frame_t, q, p, v)
        tangent = self.mode == 1
        q, p, e, v = q.copy(), p.copy(), e.copy(), v.copy(); use = np.zeros(len(ids), bool)
        for f in range(len(off) - 1):
            if not v[f]:
                continue
            c = np.arange(off[f], off[f + 1])
            good = c[(ok[c] > 0) & (ids[c] >= 0) & (ids[c] < board.shape[0])]
            if len(c) < mp or len(good) < 6:
                q[f], p[f], e[f], v[f] = [0, 0, 0, 1.0], 0.0, 0.0, 0
                continue
            X = board[ids[good], :3] / board[ids[good], 3:]
            tau = uv[good, 1] * self.line_delay; w, u = vel[f, :3], vel[f, 3:]
            Rcw = _R(q[f]).T
            R, t = refine_pose_rs(Rcw, -Rcw @ p[f], X, meas[good], tau, w, u, tangent)
            r, fr, _, _ = _errors(_rs_points(R, t, X, tau, w, u)[0], meas[good], tangent)
            inl = fr & (np.sum(r * r, 1) < thresh)
            if inl.sum() < 6:
                q[f], p[f], e[f], v[f] = [0, 0, 0, 1.0], 0.0, 0.0, 0
                continue
            if not inl.all():
                R, t = refine_pose_rs(R, t, X[inl], meas[good][inl], tau[inl], w, u, tangent)
            r = _errors(_rs_points(R, t, X[inl], tau[inl], w, u)[0], meas[good][inl], tangent)[0]
            e[f] = float(np.mean(np.linalg.norm(r, axis=1)))
            q[f] = Rotation.from_matrix(R.T).as_quat(); p[f] = -R.T @ t; v[f] = int(e[f] <= max_px)
            use[good[inl]] = True
        return q, p, e, v, use, vel, nbr

    def estimate_board_poses(self, corner_offsets, point_ids, uv, max_reproj_error=0.0, min_points=0):
        off = np.asarray(corner_offsets); ids = np.asarray(point_ids); uv = np.asarray(uv, dtype=np.float64).reshape(-1, 2)
        self._check(off)
        q, p, e, v = super().estimate_board_poses(off, ids, uv, max_reproj_error, min_points)
        if self.line_delay == 0:
            return q, p, e, v
        return self.rolling_passes(off, ids, uv, (q, p, e, v), max_reproj_error, min_points)

    def rolling_passes(self, corner_offsets, point_ids, uv, global_shutter, max_reproj_error=0.0, min_points=0):
        """The two rolling-shutter passes of estimate_board_poses from given global-shutter results (q, p, e, v) -> (q, p, e, v)"""
        off = np.asarray(corner_offsets); ids = np.asarray(point_ids); uv = np.asarray(uv, dtype=np.float64).reshape(-1, 2)
        self._check(off)
        q, p, e, v = (np.array(x, copy=True) for x in global_shutter)
        rules = self._rules(max_reproj_error, min_points)
        for _ in range(2):
            q, p, e, v, _, vel, nbr = self._rs_pass(off, ids, uv, self.board, rules, q, p, e, v)
        self.vel, self.n_static = vel, int(np.sum(nbr == 0))
        return q, p, e, v

    def optimize_board_points(self, corner_offsets, point_ids, uv, q_wc, p_wc, valid, max_reproj_error=0.0, min_points=0, min_observations=0):
        off = np.asarray(corner_offsets); ids = np.asarray(point_ids); uv = np.asarray(uv, dtype=np.float64).reshape(-1, 2)
        self._check(off)
        if self.line_delay == 0:
            return super().optimize_board_points(off, ids, uv, q_wc, p_wc, valid, max_reproj_error, min_points, min_observations)
        rules = self._rules(max_reproj_error, min_points)
        n = len(off) - 1
        q, p, v = np.array(q_wc, dtype=np.float64), np.array(p_wc, dtype=np.float64), np.array(valid, dtype=np.int32)
        q, p, e, v, use, _, _ = self._rs_pass(off, ids, uv, self.board, rules, q, p, np.zeros(n), v)
        vel, _ = view_velocities(self.frame_t, q, p, v)
        meas, ok = self._meas(uv)
        min_obs = min_observations if min_observations > 0 else 30
        view = np.repeat(np.arange(n), np.diff(off))
        take = use & (v[view] > 0)
        B = self.board.copy(); n_opt = 0
        for pt in range(B.shape[0]):
            cs = np.nonzero(take & (ids == pt))[0]
            if len(cs) <= min_obs:
                continue
            Rs = np.stack([_R(q[view[c]]).T for c in cs])
            B[pt] = np.r_[refine_point_rs(B[pt, :3] / B[pt, 3], meas[cs], Rs, p[view[cs]], uv[cs, 1] * self.line_delay, vel[view[cs], :3], vel[view[cs], 3:],
                                          self.mode == 1), 1.0]
            n_opt += 1
        q, p, e, v, _, vel, nbr = self._rs_pass(off, ids, uv, B, rules, q, p, e, v)
        self.vel, self.n_static = vel, int(np.sum(nbr == 0))
        self.board = B; self._rs_board = B
        return q, p, e, v, B, n_opt
