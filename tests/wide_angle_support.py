"""Test infrastructure of the pose step's tangent residual (ICC_POSE_ERROR_TANGENT).

- `host_math_lib()`: the product's bearing header (csrc/icc_bearing_math.cuh) compiled for the CPU (nvcc, host code only), built once per
  process into a temporary directory.
- `PoseOracle`: the oracle of icc_estimate_board_poses / icc_optimize_board_points with the same method shapes as `_capi.CApi`.  The
  normalised setting is the C++ oracle (oracle/icc_oracle.cpp); the tangent setting is restated here in NumPy, independently of the product
  header: published closed-form inverses of the camera models (Usenko et al. 2018 for DoubleSphere, Khomutenko et al. 2016 for
  ExtendedUnified), its own tangent basis, a left-increment Levenberg-Marquardt and an SVD homography start.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from openimucameracalibrator_b200 import camera_models as cm

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
HUBER = 1.345


def host_math_lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_wide_angle_"), "libwide_angle_host_math.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "wide_angle", "bearing_host_math.cu")])
        _LIB = ctypes.CDLL(out)
    return _LIB


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def product_bearings(model, k, uv):
    """(xyz[n,3], ok[n]) from the product's unproject_bearing on the CPU."""
    uv = np.ascontiguousarray(uv, dtype=np.float64).reshape(-1, 2); k = np.ascontiguousarray(k, dtype=np.float64)
    n = uv.shape[0]; xyz = np.zeros((n, 3)); ok = np.zeros(n, dtype=np.int32)
    host_math_lib().wa_unproject_bearings(int(model), _dp(k), n, _dp(uv), _dp(xyz), ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    return xyz, ok


def product_tangent_error(b, q_xyzw, X, t):
    """-> (r[2], front, J[2,6] pose Jacobian for the right increment, P[2,3] board-point Jacobian) of the product header."""
    a = [np.ascontiguousarray(v, dtype=np.float64) for v in (b, q_xyzw, X, t)]
    r = np.zeros(2); J = np.zeros(12); P = np.zeros(6)
    front = host_math_lib().wa_tangent_error(*[_dp(v) for v in a], _dp(r), _dp(J), _dp(P))
    return r, bool(front), J.reshape(2, 6), P.reshape(2, 3)


def product_tangent_basis(b):
    b = np.ascontiguousarray(b, dtype=np.float64); e1 = np.zeros(3); e2 = np.zeros(3)
    host_math_lib().wa_tangent_basis(_dp(b), _dp(e1), _dp(e2))
    return e1, e2


# ---- closed-form inverses of the seven models ----------------------------------------------------------------------------------------
def _skew_inverse(k, uv):
    dy = (uv[:, 1] - k[4]) / (k[0] * k[1])
    return (uv[:, 0] - k[3] - k[2] * dy) / k[0], dy


def _radial_inverse(rd, poly, dpoly):
    """ru with ru * poly(ru^2) = rd by Newton from ru = rd."""
    ru = rd.copy()
    for _ in range(100):
        ru = ru - (ru * poly(ru * ru) - rd) / dpoly(ru * ru)
    return ru


def oracle_bearings(model, k, uv):
    """Unit rays of an (n, 2) pixel array -> (xyz[n,3], ok[n]); ok = in the inverse's domain and reprojecting within 1e-6 px."""
    k = np.asarray(k, dtype=np.float64); uv = np.asarray(uv, dtype=np.float64).reshape(-1, 2)
    n = uv.shape[0]; ok = np.ones(n, bool)
    if model in (cm.PINHOLE, cm.PINHOLE_RADIAL_TANGENTIAL):
        dx, dy = _skew_inverse(k, uv)
        if model == cm.PINHOLE:
            rd = np.hypot(dx, dy)
            ru = _radial_inverse(rd, lambda s: 1 + s * (k[5] + k[6] * s), lambda s: 1 + 3 * k[5] * s + 5 * k[6] * s * s)
            sc = np.where(rd > 0, ru / np.where(rd > 0, rd, 1.0), 1.0)
            x, y = dx * sc, dy * sc
        else:
            x, y = dx.copy(), dy.copy()
            k1, k2, k3, t1, t2 = k[5:10]
            for _ in range(100):
                r2 = x * x + y * y; d = 1 + r2 * (k1 + r2 * (k2 + r2 * k3)); dd = k1 + r2 * (2 * k2 + 3 * k3 * r2)
                fx = x * d + 2 * t1 * x * y + t2 * (r2 + 2 * x * x) - dx
                fy = y * d + 2 * t2 * x * y + t1 * (r2 + 2 * y * y) - dy
                a = d + 2 * x * x * dd + 2 * t1 * y + 6 * t2 * x; b = 2 * x * y * dd + 2 * t1 * x + 2 * t2 * y
                c = 2 * x * y * dd + 2 * t2 * y + 2 * t1 * x; e = d + 2 * y * y * dd + 2 * t2 * x + 6 * t1 * y
                det = a * e - b * c
                x, y = x - (e * fx - b * fy) / det, y - (-c * fx + a * fy) / det
        xyz = np.stack([x, y, np.ones(n)], -1)
    elif model == cm.FOV:
        mx, my = (uv[:, 0] - k[2]) / k[0], (uv[:, 1] - k[3]) / (k[0] * k[1])
        rd = np.hypot(mx, my); om = k[4]
        if om * om < 1e-10:
            sc = np.ones(n)
        else:
            ru = np.tan(rd * om) / (2 * np.tan(0.5 * om))
            sc = np.where(rd > 1e-12, ru / np.where(rd > 1e-12, rd, 1.0), om / (2 * np.tan(0.5 * om)))
        xyz = np.stack([mx * sc, my * sc, np.ones(n)], -1)
    elif model == cm.DIVISION_UNDISTORTION:
        ud, vd = uv[:, 0] - k[2], uv[:, 1] - k[3]
        s = 1.0 / (1.0 + k[4] * (ud * ud + vd * vd))
        xyz = np.stack([ud * s / k[0], vd * s / (k[0] * k[1]), np.ones(n)], -1)
    elif model == cm.FISHEYE:
        dx, dy = _skew_inverse(k, uv)
        thd = np.hypot(dx, dy)
        th = _radial_inverse(thd, lambda s: 1 + s * (k[5] + s * (k[6] + s * (k[7] + s * k[8]))),
                             lambda s: 1 + s * (3 * k[5] + s * (5 * k[6] + s * (7 * k[7] + s * 9 * k[8]))))
        ok &= th < np.pi / 2
        sc = np.where(thd > 0, np.sin(th) / np.where(thd > 0, thd, 1.0), 1.0)
        xyz = np.stack([dx * sc, dy * sc, np.cos(th)], -1)
    elif model == cm.DOUBLE_SPHERE:
        mx, my = _skew_inverse(k, uv)
        xi, al = k[5], k[6]
        r2 = mx * mx + my * my
        arg = 1 - (2 * al - 1) * r2
        ok &= arg >= 0
        mz = (1 - al * al * r2) / (al * np.sqrt(np.maximum(arg, 0)) + 1 - al)
        f = (mz * xi + np.sqrt(np.maximum(mz * mz + (1 - xi * xi) * r2, 0))) / (mz * mz + r2)
        xyz = np.stack([f * mx, f * my, f * mz - xi], -1)
    elif model == cm.EXTENDED_UNIFIED:
        mx, my = _skew_inverse(k, uv)
        al, be = k[5], k[6]
        r2 = mx * mx + my * my
        arg = 1 - (2 * al - 1) * be * r2
        ok &= arg >= 0
        mz = (1 - be * al * al * r2) / (al * np.sqrt(np.maximum(arg, 0)) + 1 - al)
        xyz = np.stack([mx, my, mz], -1)
    else:
        raise ValueError(model)
    xyz = xyz / np.linalg.norm(xyz, axis=1, keepdims=True)
    px, valid = cm.project(model, k, xyz)
    ok &= valid & (np.linalg.norm(px - uv, axis=1) < 1e-6) & np.isfinite(xyz).all(1)
    return xyz, ok.astype(np.int32)


# ---- tangent-mode pose and board-point steps -----------------------------------------------------------------------------------------
def oracle_basis(b):
    """A tangent basis of its own (any orthonormal one gives the same |r|): e1 = normalise(a x b) with a the axis least aligned with b."""
    a = np.where((np.abs(b[:, 0]) < 0.6)[:, None], np.array([1.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]))
    e1 = np.cross(a, b); e1 /= np.linalg.norm(e1, axis=1, keepdims=True)
    return e1, np.cross(b, e1)


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def _exp(w):
    th = np.linalg.norm(w)
    K = _skew(w)
    if th < 1e-12:
        return np.eye(3) + K + 0.5 * K @ K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def _residuals(R, t, X, b, e1, e2):
    d = X @ R.T + t
    s = np.einsum("ij,ij->i", b, d)
    r = np.stack([np.einsum("ij,ij->i", e1, d), np.einsum("ij,ij->i", e2, d)], -1) / s[:, None]
    return d, s, r


def _huber_cost(r, s):
    rn = np.linalg.norm(r, axis=1)
    return float(np.sum(np.where(rn <= HUBER, 0.5 * rn * rn, HUBER * rn - 0.5 * HUBER * HUBER)) + 1e6 * np.sum(~(s > 0)))


def refine_pose(R, t, X, b, iters=200):
    """Levenberg-Marquardt on the Huber(1.345) tangent cost, left increment R <- exp(w) R, t <- t + dt, to a 1e-16 relative stall."""
    e1, e2 = oracle_basis(b)
    d, s, r = _residuals(R, t, X, b, e1, e2)
    cost = _huber_cost(r, s); lam = 1e-3
    for _ in range(iters):
        rn = np.linalg.norm(r, axis=1); w = np.where(rn <= HUBER, 1.0, HUBER / np.maximum(rn, 1e-300))
        # dr/dd = (e - r b) / s ; dd/dw = -[d - t]x = -[R X]x ; dd/dt = I
        A0 = (e1 - r[:, :1] * b) / s[:, None]; A1 = (e2 - r[:, 1:] * b) / s[:, None]
        RX = d - t
        J = np.concatenate([np.concatenate([np.cross(RX, A0), A0], 1)[:, None], np.concatenate([np.cross(RX, A1), A1], 1)[:, None]], 1)   # n x 2 x 6
        fr = s > 0
        Jw = J[fr] * np.sqrt(w[fr])[:, None, None]; rw = r[fr] * np.sqrt(w[fr])[:, None]
        H = np.einsum("nij,nik->jk", Jw, Jw); g = np.einsum("nij,ni->j", Jw, rw)
        stepped = False
        while lam < 1e16:
            dx = np.linalg.solve(H + lam * np.diag(np.diag(H) + 1e-12), -g)
            Rn = _exp(dx[:3]) @ R; tn = t + dx[3:]
            dn, sn, rn2 = _residuals(Rn, tn, X, b, e1, e2)
            cn = _huber_cost(rn2, sn)
            if cn < cost:
                dec = cost - cn
                R, t, d, s, r, cost = Rn, tn, dn, sn, rn2, cn
                lam = max(lam * 0.1, 1e-14); stepped = True
                break
            lam *= 10
        if not stepped or dec <= 1e-16 * cost or dx @ dx < 1e-30:
            break
    U, _, Vt = np.linalg.svd(R)
    return U @ Vt, t


def _homography_start(X, b):
    """Rotate the bearings so that their mean is +z, DLT homography (SVD, Hartley-normalised) of those within 80 degrees, back to R_cw, t."""
    m = b.sum(0); m /= np.linalg.norm(m)
    a = np.array([1.0, 0.0, 0.0]) if abs(m[0]) < 0.6 else np.array([0.0, 1.0, 0.0])
    u = np.cross(a, m); u /= np.linalg.norm(u)
    Rm = np.stack([u, np.cross(m, u), m])                         # rows: R_m m = e_z
    bm = b @ Rm.T
    near = bm[:, 2] > np.cos(np.radians(80))
    if near.sum() < 6:
        return None
    xy = bm[near, :2] / bm[near, 2:]; P = X[near, :2]
    def norm(p):
        c = p.mean(0); s = np.sqrt(2) / np.mean(np.linalg.norm(p - c, axis=1))
        return np.array([[s, 0, -s * c[0]], [0, s, -s * c[1]], [0, 0, 1]])
    Tb, Ti = norm(P), norm(xy)
    Ph = np.c_[P, np.ones(len(P))] @ Tb.T; xh = np.c_[xy, np.ones(len(xy))] @ Ti.T
    A = []
    for (X0, Y0, _), (x0, y0, _) in zip(Ph, xh):
        A.append([X0, Y0, 1, 0, 0, 0, -x0 * X0, -x0 * Y0, -x0]); A.append([0, 0, 0, X0, Y0, 1, -y0 * X0, -y0 * Y0, -y0])
    Hn = np.linalg.svd(np.array(A))[2][-1].reshape(3, 3)
    Hm = np.linalg.inv(Ti) @ Hn @ Tb
    s = 2.0 / (np.linalg.norm(Hm[:, 0]) + np.linalg.norm(Hm[:, 1]))
    if Hm[2, 2] * s < 0:
        s = -s
    r1, r2, tm = s * Hm[:, 0], s * Hm[:, 1], s * Hm[:, 2]
    U, _, Vt = np.linalg.svd(np.stack([r1, r2, np.cross(r1, r2)], 1))
    Rr = U @ Vt
    return Rm.T @ Rr, Rm.T @ tm


def _fail():
    return np.array([0.0, 0.0, 0.0, 1.0]), np.zeros(3), 0.0, 0


def _rot_to_quat(R):
    from scipy.spatial.transform import Rotation
    return Rotation.from_matrix(R).as_quat()                   # x, y, z, w


def _quat_to_rot(q):
    from scipy.spatial.transform import Rotation
    return Rotation.from_quat(q).as_matrix()


def tangent_view(X, b, n_all, min_points, thresh_sq, max_err, start=None):
    """One view: X[n,3] board points, b[n,3] bearings of the usable corners (n_all = every corner of the view, the min_points rule).
    start = (R_cw, t) for a refinement-only pass.  -> (q_wc, p_wc, mean tangent error, valid, inlier mask)."""
    none = np.zeros(len(b), bool)
    if n_all < min_points or len(b) < 6:
        return (*_fail(), none)
    if start is None:
        z = X[:, 2].mean(); dB = np.mean(np.linalg.norm(X[:, :2] - X[:, :2].mean(0), axis=1))
        if np.abs(X[:, 2] - z).max() > 0.05 * dB:
            return (*_fail(), none)
        st = _homography_start(np.c_[X[:, :2], X[:, 2] - z], b)
        if st is None:
            return (*_fail(), none)
        R, t = st; t = t - z * R[:, 2]
    else:
        R, t = start
    R, t = refine_pose(R, t, X, b)
    e1, e2 = oracle_basis(b)
    _, s, r = _residuals(R, t, X, b, e1, e2)
    inl = (s > 0) & (np.sum(r * r, 1) < thresh_sq)
    if inl.sum() < 6:
        return (*_fail(), none)
    if not inl.all():
        R, t = refine_pose(R, t, X[inl], b[inl])
        _, s, r = _residuals(R, t, X[inl], b[inl], e1[inl], e2[inl])
    e = float(np.mean(np.linalg.norm(r, axis=1)))
    return _rot_to_quat(R.T), -R.T @ t, e, int(e <= max_err), inl


def refine_point(X, bs, Rs, cs):
    """Board point X with constant cameras (R_cw, centre c) against bearings bs: LM on the Huber tangent cost."""
    e1, e2 = oracle_basis(bs)
    def res(Xp):
        d = np.einsum("nij,nj->ni", Rs, Xp - cs); s = np.einsum("ij,ij->i", bs, d)
        return d, s, np.stack([np.einsum("ij,ij->i", e1, d), np.einsum("ij,ij->i", e2, d)], -1) / s[:, None]
    d, s, r = res(X); cost = _huber_cost(r, s); lam = 1e-3
    for _ in range(200):
        rn = np.linalg.norm(r, axis=1); w = np.where(rn <= HUBER, 1.0, HUBER / np.maximum(rn, 1e-300))
        A0 = (e1 - r[:, :1] * bs) / s[:, None]; A1 = (e2 - r[:, 1:] * bs) / s[:, None]
        J = np.stack([np.einsum("ni,nij->nj", A0, Rs), np.einsum("ni,nij->nj", A1, Rs)], 1)
        fr = s > 0
        Jw = J[fr] * np.sqrt(w[fr])[:, None, None]; rw = r[fr] * np.sqrt(w[fr])[:, None]
        H = np.einsum("nij,nik->jk", Jw, Jw); g = np.einsum("nij,ni->j", Jw, rw)
        stepped = False
        while lam < 1e16:
            dx = np.linalg.solve(H + lam * np.diag(np.diag(H) + 1e-12), -g)
            dn, sn, rn2 = res(X + dx); cn = _huber_cost(rn2, sn)
            if cn < cost:
                dec = cost - cn; X, d, s, r, cost = X + dx, dn, sn, rn2, cn; lam = max(lam * 0.1, 1e-14); stepped = True
                break
            lam *= 10
        if not stepped or dec <= 1e-16 * cost or dx @ dx < 1e-32:
            break
    return X


class PoseOracle:
    """icc_estimate_board_poses / icc_optimize_board_points oracle with icc_set_pose_error: normalised = the C++ oracle, tangent = NumPy."""

    def __init__(self):
        from oracle_api import new_oracle
        self.cpp = new_oracle(); self.mode = 0

    def set_camera(self, model, k, W, H):
        self.model, self.k, self.W, self.H = model, np.asarray(k, dtype=np.float64), W, H
        self.cpp.set_camera(model, k, W, H)

    def set_board_points(self, xyzw):
        self.board = np.array(xyzw, dtype=np.float64).reshape(-1, 4)
        self.cpp.set_board_points(xyzw)

    def set_pose_error(self, mode):
        from openimucameracalibrator_b200 import _capi as capi
        mode = capi.POSE_ERRORS[mode] if isinstance(mode, str) else int(mode)
        if mode not in (0, 1):
            raise ValueError(mode)
        self.mode = mode

    def get_board_points(self):
        return self.board.copy() if self.mode == 1 else self.cpp.get_board_points()

    def pixels_to_bearings(self, uv):
        return oracle_bearings(self.model, self.k, uv)

    def _rules(self, max_reproj_error, min_points):
        max_px = max_reproj_error if max_reproj_error > 0 else 0.004 * self.H
        thresh = max_px / np.hypot(self.W, self.H) if self.W > 0 and self.H > 0 else 1e-3
        return (min_points if min_points > 0 else 8), thresh, max_px

    def _views(self, off, ids, uv, board, max_reproj_error, min_points, starts=None):
        b, ok = oracle_bearings(self.model, self.k, uv)
        mp, thresh, max_px = self._rules(max_reproj_error, min_points)
        n = len(off) - 1
        q = np.zeros((n, 4)); p = np.zeros((n, 3)); e = np.zeros(n); v = np.zeros(n, np.int32); use = np.zeros(len(ids), bool)
        q[:, 3] = 1
        for f in range(n):
            c = np.arange(off[f], off[f + 1])
            good = c[(ok[c] > 0) & (ids[c] >= 0) & (ids[c] < board.shape[0])]
            X = board[ids[good], :3] / board[ids[good], 3:]
            start = None
            if starts is not None:
                sq, sp, sv = starts
                if not sv[f]:
                    q[f], p[f] = sq[f], sp[f]
                    continue
                R = _quat_to_rot(sq[f]).T; start = (R, -R @ sp[f])
            q[f], p[f], e[f], v[f], inl = tangent_view(X, b[good], len(c), mp, thresh, max_px, start)
            use[good[inl]] = True
        return q, p, e, v, use, b

    def estimate_board_poses(self, corner_offsets, point_ids, uv, max_reproj_error=0.0, min_points=0):
        if self.mode == 0:
            return self.cpp.estimate_board_poses(corner_offsets, point_ids, uv, max_reproj_error, min_points)
        off = np.asarray(corner_offsets); ids = np.asarray(point_ids)
        q, p, e, v, _, _ = self._views(off, ids, np.asarray(uv, dtype=np.float64).reshape(-1, 2), self.board, max_reproj_error, min_points)
        return q, p, e, v

    def optimize_board_points(self, corner_offsets, point_ids, uv, q_wc, p_wc, valid, max_reproj_error=0.0, min_points=0, min_observations=0):
        if self.mode == 0:
            return self.cpp.optimize_board_points(corner_offsets, point_ids, uv, q_wc, p_wc, valid, max_reproj_error, min_points, min_observations)
        off = np.asarray(corner_offsets); ids = np.asarray(point_ids); uv = np.asarray(uv, dtype=np.float64).reshape(-1, 2)
        starts = (np.asarray(q_wc, dtype=np.float64), np.asarray(p_wc, dtype=np.float64), np.asarray(valid))
        q, p, e, v, use, b = self._views(off, ids, uv, self.board, max_reproj_error, min_points, starts)
        min_obs = min_observations if min_observations > 0 else 30
        view = np.repeat(np.arange(len(off) - 1), np.diff(off))
        take = use & (v[view] > 0)
        B = self.board.copy(); n_opt = 0
        for pt in range(B.shape[0]):
            cs = np.nonzero(take & (ids == pt))[0]
            if len(cs) <= min_obs:
                continue
            Rs = np.stack([_quat_to_rot(q[view[c]]).T for c in cs]); cc = p[view[cs]]
            B[pt] = np.r_[refine_point(B[pt, :3] / B[pt, 3], b[cs], Rs, cc), 1.0]; n_opt += 1
        q, p, e, v, _, _ = self._views(off, ids, uv, B, max_reproj_error, min_points, (q, p, v))
        self.board = B
        return q, p, e, v, B, n_opt
