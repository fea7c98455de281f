"""NumPy camera projections used by the synthetic-data generator (host-side, FP64).

Third, independent statement of the Theia camera-model equations that the reference dispatches at
include/OpenCameraCalibrator/basalt_spline/ceres_calib_split_residuals.h:366-389 (the device statement lives in
csrc/icc_camera.cuh, the autodiff statement in oracle/oracle_math.hpp).  Model ids are theia::CameraIntrinsicsModelType
values; JSON names follow src/io/read_camera_calibration.cc:59-116.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

PINHOLE, PINHOLE_RADIAL_TANGENTIAL, FISHEYE, FOV, DIVISION_UNDISTORTION, DOUBLE_SPHERE, EXTENDED_UNIFIED = range(7)
OMNI_RADIAL_TANGENTIAL = 7   # extension without a Theia counterpart: Kalibr's omni-radtan
SCARAMUZZA = 8               # extension without a Theia counterpart: Scaramuzza's omnidirectional polynomial model (OCamCalib)
PINHOLE_RATIONAL = 9         # extension without a Theia counterpart: OpenCV's rational polynomial model (k1..k6, p1, p2)
FISHEYE_RADIAL_TANGENTIAL = 10   # extension without a Theia counterpart: Kannala-Brandt with k1..k6 and tangential t1, t2 (Fisheye62)


class CameraLayout(NamedTuple):
    """One camera model in the camera JSON and the tools' printed summary.  The same table, row for row, is kCameraLayouts in
    csrc/icc_cli_common.hpp."""
    name: str          # `intrinsic_type`
    id: int            # ICC_CAM_* / theia::CameraIntrinsicsModelType
    num_params: int
    keys: dict         # JSON key -> Theia index of every intrinsic the file carries, in file order; `skew` only where index 2 is the skew
    printed: dict      # label -> index of the model's PrintResult line, "" for an unlabelled value; empty when the tools print none


_AFFINE = {"focal_length": 0, "aspect_ratio": 1, "skew": 2, "principal_pt_x": 3, "principal_pt_y": 4}
_AFFINE_NOSKEW = {"focal_length": 0, "aspect_ratio": 1, "principal_pt_x": 2, "principal_pt_y": 3}
CAMERAS = {c.id: c for c in (
    CameraLayout("PINHOLE", PINHOLE, 7, _AFFINE, {}),
    CameraLayout("PINHOLE_RADIAL_TANGENTIAL", PINHOLE_RADIAL_TANGENTIAL, 10,
                 dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, tangential_distortion_1=8, tangential_distortion_2=9), {}),
    CameraLayout("FISHEYE", FISHEYE, 9, dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, radial_distortion_4=8),
                 {"Radial distortion 1": 5, "Radial distortion 2": 6, "Radial distortion 3": 7, "Radial distortion 4": 8}),
    CameraLayout("FOV", FOV, 5, dict(_AFFINE_NOSKEW, radial_distortion_1=4), {}),
    CameraLayout("DIVISION_UNDISTORTION", DIVISION_UNDISTORTION, 5, dict(_AFFINE_NOSKEW, div_undist_distortion=4), {"Distortion": 4}),
    CameraLayout("DOUBLE_SPHERE", DOUBLE_SPHERE, 7, dict(_AFFINE, xi=5, alpha=6), {"XI": 5, "ALPHA": 6}),
    CameraLayout("EXTENDED_UNIFIED", EXTENDED_UNIFIED, 7, dict(_AFFINE, alpha=5, beta=6), {"": 5, "BETA": 6}),
    CameraLayout("OMNI_RADIAL_TANGENTIAL", OMNI_RADIAL_TANGENTIAL, 10,
                 dict(_AFFINE, xi=5, radial_distortion_1=6, radial_distortion_2=7, tangential_distortion_1=8, tangential_distortion_2=9),
                 {"XI": 5, "Radial distortion 1": 6, "Radial distortion 2": 7, "Tangential distortion 1": 8, "Tangential distortion 2": 9}),
    CameraLayout("SCARAMUZZA", SCARAMUZZA, 9,   # index 2 is the stretch e, not a skew
                 dict(focal_length=0, aspect_ratio=1, principal_pt_x=3, principal_pt_y=4, stretch_d=8, stretch_e=2, polynomial_a2=5, polynomial_a3=6, polynomial_a4=7),
                 {"A2": 5, "A3": 6, "A4": 7, "Stretch c": 1, "d": 8, "e": 2}),
    CameraLayout("PINHOLE_RATIONAL", PINHOLE_RATIONAL, 13, dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, tangential_distortion_1=8,
                                                                tangential_distortion_2=9, radial_distortion_4=10, radial_distortion_5=11, radial_distortion_6=12),
                 {"Radial distortion 1": 5, "Radial distortion 2": 6, "Radial distortion 3": 7, "Radial distortion 4": 10, "Radial distortion 5": 11,
                  "Radial distortion 6": 12, "Tangential distortion 1": 8, "Tangential distortion 2": 9}),
    CameraLayout("FISHEYE_RADIAL_TANGENTIAL", FISHEYE_RADIAL_TANGENTIAL, 13,
                 dict(_AFFINE, radial_distortion_1=5, radial_distortion_2=6, radial_distortion_3=7, radial_distortion_4=8, radial_distortion_5=9,
                      radial_distortion_6=10, tangential_distortion_1=11, tangential_distortion_2=12),
                 {"Radial distortion 1": 5, "Radial distortion 2": 6, "Radial distortion 3": 7, "Radial distortion 4": 8, "Radial distortion 5": 9,
                  "Radial distortion 6": 10, "Tangential distortion 1": 11, "Tangential distortion 2": 12}),
)}
MODEL_NAMES = {m: c.name for m, c in CAMERAS.items()}
MODEL_IDS = {c.name: m for m, c in CAMERAS.items()}
NUM_PARAMS = {m: c.num_params for m, c in CAMERAS.items()}
MAX_INTRINSICS = 13   # ICC_MAX_INTRINSICS: the longest intrinsic vector


def _affine_skew(k, dx, dy):
    return np.stack([k[0] * dx + k[2] * dy + k[3], k[0] * k[1] * dy + k[4]], axis=-1)


def _unified_w(alpha):
    return (1.0 - alpha) / alpha if alpha > 0.5 else alpha / (1.0 - alpha)


def scaramuzza_F(k, rho):
    """F(rho) = a0 + a2 rho^2 + a3 rho^3 + a4 rho^4 of SCARAMUZZA's [a0, c, e, cx, cy, a2, a3, a4, d]"""
    return k[0] + rho * rho * (k[5] + rho * (k[6] + rho * k[7]))


def scaramuzza_rho_max(k) -> float:
    """First stationary point of F(rho) / rho: the smallest positive root of 3 a4 rho^4 + 2 a3 rho^3 + a2 rho^2 - a0 (np.roots, polished by
    Newton's method), inf when there is none."""
    a0, a2, a3, a4 = (float(k[i]) for i in (0, 5, 6, 7))
    roots = np.roots([3.0 * a4, 2.0 * a3, a2, 0.0, -a0])
    pos = roots.real[(np.abs(roots.imag) <= 1e-8 * np.abs(roots)) & (roots.real > 0.0)]
    if pos.size == 0:
        return np.inf
    x = float(pos.min())
    for _ in range(4):
        dq = x * (2.0 * a2 + x * (6.0 * a3 + 12.0 * a4 * x))
        if dq != 0.0:
            x -= (x * x * (a2 + x * (2.0 * a3 + 3.0 * a4 * x)) - a0) / dq
    return x


def scaramuzza_scale(k, r, z):
    """(s, valid): the projection's scale s (sensor point = s (x, y)), the smallest positive root of a0 - z s + a2 (r s)^2 + a3 (r s)^3 +
    a4 (r s)^4 for points at distance r from the optical axis and depth z, by bisection and Newton's method over whole arrays.  A point is
    valid iff z / r > F(rho_max) / rho_max (z > 0 on the axis); with rho_max = inf that bound is 0 for a constant F and -inf otherwise."""
    k = np.asarray(k, dtype=np.float64)
    r, z = np.broadcast_arrays(np.asarray(r, dtype=np.float64), np.asarray(z, dtype=np.float64))
    a0, a2, a3, a4 = k[0], k[5], k[6], k[7]
    rmax = scaramuzza_rho_max(k)
    if np.isfinite(rmax):
        valid = z * rmax > r * scaramuzza_F(k, rmax)
    elif a2 == 0.0 and a3 == 0.0 and a4 == 0.0:
        valid = z > 0.0
    else:
        valid = (z > 0.0) | (r > 0.0)
    valid = valid & (a0 > 0.0)
    s = np.zeros(r.shape)
    if not valid.any():
        return s, valid
    rv, zv = r[valid], z[valid]

    def h(x, i):    # -G(x) and -G_s(x) of the points i, increasing along the branch
        rho = rv[i] * x
        return zv[i] * x - scaramuzza_F(k, rho), zv[i] - rv[i] * rho * (2.0 * a2 + rho * (3.0 * a3 + 4.0 * a4 * rho))

    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        cap = np.where(rv > 0.0, rmax / rv, np.inf)
        lo, hi = np.zeros(rv.shape), np.minimum(a0 / np.hypot(rv, zv), cap)
        i = np.arange(rv.size)
        for _ in range(1100):              # grow the bracket until -G(hi) >= 0 or hi reaches rho_max / r
            i = i[(h(hi[i], i)[0] < 0.0) & (hi[i] < cap[i])]
            if i.size == 0:
                break
            lo[i] = hi[i]
            hi[i] = np.minimum(2.0 * hi[i], cap[i])
        x = 0.5 * (lo + hi)
        i = np.arange(rv.size)
        for _ in range(200):               # Newton's method, bisection where a step leaves the bracket, until the step is an ulp or two
            xi, li, hi_ = x[i], lo[i], hi[i]
            f, df = h(xi, i)
            li = np.where(f < 0.0, xi, li)
            hi_ = np.where(f > 0.0, xi, hi_)
            xn = xi - f / df
            xn = np.where((xn > li) & (xn < hi_), xn, 0.5 * (li + hi_))
            xn = np.where(f == 0.0, xi, xn)
            x[i], lo[i], hi[i] = xn, li, hi_
            i = i[np.abs(xn - xi) > 2.5e-16 * np.abs(xn)]
            if i.size == 0:
                break
    s[valid] = x
    return s, valid


def rational_s_max(k) -> float:
    """PINHOLE_RATIONAL's [f, ar, skew, cx, cy, k1, k2, k3, t1, t2, k4, k5, k6]: the first s = xn^2 + yn^2 > 0 at which the radial map
    r R(r^2), R = N / M, stops increasing: the smallest positive real root of M or of h = N M + 2 s (N' M - N M') (np.roots), inf when
    there is none."""
    k = np.asarray(k, dtype=np.float64)
    n = np.array([1.0, k[5], k[6], k[7]])                # ascending powers of s
    m = np.array([1.0, k[10], k[11], k[12]])
    nm = np.convolve(n, m)
    dn, dm = n[1:] * np.arange(1, 4), m[1:] * np.arange(1, 4)
    h = nm.copy()
    h[1:] += 2.0 * (np.convolve(dn, m) - np.convolve(n, dm))   # s (N' M - N M')
    best = np.inf
    for c in (m, h):
        c = np.trim_zeros(c, "b")
        if c.size < 2:
            continue
        roots = np.roots(c[::-1])
        pos = roots.real[(np.abs(roots.imag) <= 1e-9 * np.maximum(np.abs(roots), 1.0)) & (roots.real > 0.0)]
        if pos.size:
            best = min(best, float(pos.min()))
    return best


def rational_distort(k, xn, yn):
    """PINHOLE_RATIONAL's distorted normalised point (dx, dy) of (xn, yn)"""
    s = xn * xn + yn * yn
    R = (1.0 + s * (k[5] + s * (k[6] + s * k[7]))) / (1.0 + s * (k[10] + s * (k[11] + s * k[12])))
    return (xn * R + 2.0 * k[8] * xn * yn + k[9] * (s + 2.0 * xn * xn),
            yn * R + k[8] * (s + 2.0 * yn * yn) + 2.0 * k[9] * xn * yn)


def rational_unproject(k, uv):
    """PINHOLE_RATIONAL: (xn, yn) = (x / z, y / z) of pixels uv (..., 2) and ok (...,): the skewed affine inverted, then damped Newton's
    method on the distortion over whole arrays (Jacobian by central differences), started at the distorted point pulled inside the domain;
    ok iff the point converged to 1e-12 of the distorted point and lies inside the domain s < s_max."""
    k = np.asarray(k, dtype=np.float64)
    uv = np.asarray(uv, dtype=np.float64)
    dy = (uv[..., 1] - k[4]) / (k[0] * k[1])
    dx = (uv[..., 0] - k[3] - k[2] * dy) / k[0]
    smax = rational_s_max(k)
    shrink = np.where(dx * dx + dy * dy < 0.5 * smax, 1.0, np.sqrt(0.5 * smax / np.maximum(dx * dx + dy * dy, 1e-300)))
    x, y = dx * shrink, dy * shrink                      # a start inside the domain

    def err(x, y):
        fx, fy = rational_distort(k, x, y)
        return np.where(x * x + y * y < smax, np.hypot(fx - dx, fy - dy), np.inf), fx - dx, fy - dy

    with np.errstate(all="ignore"):
        for _ in range(100):                             # Newton's method, each step halved until it stays inside and improves
            e, ex, ey = err(x, y)
            h = 1e-7 * np.maximum(1.0, np.hypot(x, y))
            ax = (np.array(rational_distort(k, x + h, y)) - np.array(rational_distort(k, x - h, y))) / (2.0 * h)
            ay = (np.array(rational_distort(k, x, y + h)) - np.array(rational_distort(k, x, y - h))) / (2.0 * h)
            det = ax[0] * ay[1] - ay[0] * ax[1]
            sx, sy = -(ay[1] * ex - ay[0] * ey) / det, -(-ax[1] * ex + ax[0] * ey) / det
            t = np.ones_like(x)
            for _ in range(40):
                bad = ~(err(x + t * sx, y + t * sy)[0] <= e)
                if not bad.any():
                    break
                t = np.where(bad, 0.5 * t, t)
            moved = err(x + t * sx, y + t * sy)[0] <= e
            x, y = np.where(moved, x + t * sx, x), np.where(moved, y + t * sy, y)
        fx, fy = rational_distort(k, x, y)
        ok = (np.hypot(fx - dx, fy - dy) <= 1e-12 * np.maximum(1.0, np.hypot(dx, dy))) & (x * x + y * y < smax)
    return np.stack([x, y], axis=-1), ok


def fisheye_radtan_theta_max(k) -> float:
    """FISHEYE_RADIAL_TANGENTIAL's [f, ar, skew, cx, cy, k1, k2, k3, k4, k5, k6, t1, t2]: the first theta > 0 at which theta_d = theta (1 +
    k1 theta^2 + ... + k6 theta^12) stops increasing, i.e. sqrt of the smallest positive real root t of d theta_d / d theta = 1 + 3 k1 t +
    5 k2 t^2 + ... + 13 k6 t^6 (np.roots), inf when there is none."""
    k = np.asarray(k, dtype=np.float64)
    q = np.trim_zeros(np.concatenate([[1.0], np.arange(3, 15, 2) * k[5:11]]), "b")
    if q.size < 2:
        return np.inf
    roots = np.roots(q[::-1])
    pos = roots.real[(np.abs(roots.imag) <= 1e-9 * np.maximum(np.abs(roots), 1.0)) & (roots.real > 0.0)]
    return float(np.sqrt(pos.min())) if pos.size else np.inf


def fisheye_radtan_distort(k, x, y, z):
    """FISHEYE_RADIAL_TANGENTIAL's distorted point (dx, dy) of camera-frame points (x, y, z), z > 0: the radial stage (xr, yr) = (theta_d / r)
    (x, y) ((x, y) / z on the axis), then the tangential terms of PINHOLE_RADIAL_TANGENTIAL"""
    r = np.hypot(x, y)
    th = np.arctan2(r, z); t = th * th
    P = 1.0 + t * (k[5] + t * (k[6] + t * (k[7] + t * (k[8] + t * (k[9] + t * k[10])))))
    with np.errstate(divide="ignore", invalid="ignore"):
        g = np.where(r > 0.0, th * P / np.where(r > 0.0, r, 1.0), 1.0 / z)
    xr, yr = g * x, g * y
    s = xr * xr + yr * yr
    return (xr + 2.0 * k[11] * xr * yr + k[12] * (s + 2.0 * xr * xr),
            yr + k[11] * (s + 2.0 * yr * yr) + 2.0 * k[12] * xr * yr)


def fisheye_radtan_unproject(k, uv):
    """FISHEYE_RADIAL_TANGENTIAL: (xn, yn) = (x / z, y / z) of pixels uv (..., 2) and ok (...,): the skewed affine inverted, then damped
    Newton's method on the normalised plane over whole arrays (Jacobian by central differences), started at the equidistant reading of the
    distorted point; ok iff the point converged to 1e-12 of the distorted point and its ray lies inside the domain theta < theta_max."""
    k = np.asarray(k, dtype=np.float64)
    uv = np.asarray(uv, dtype=np.float64)
    dy = (uv[..., 1] - k[4]) / (k[0] * k[1])
    dx = (uv[..., 0] - k[3] - k[2] * dy) / k[0]
    thmax = min(fisheye_radtan_theta_max(k), 0.5 * np.pi)
    rd = np.hypot(dx, dy)
    th0 = np.minimum(rd, 0.9 * thmax)
    with np.errstate(divide="ignore", invalid="ignore"):
        sc = np.where(rd > 0.0, np.tan(th0) / np.where(rd > 0.0, rd, 1.0), 1.0)
    x, y = dx * sc, dy * sc                                 # a start inside the domain

    def err(x, y):
        fx, fy = fisheye_radtan_distort(k, x, y, 1.0)
        return np.where(np.arctan(np.hypot(x, y)) < thmax, np.hypot(fx - dx, fy - dy), np.inf), fx - dx, fy - dy

    with np.errstate(all="ignore"):
        for _ in range(100):                                 # Newton's method, each step halved until it stays inside and improves
            e, ex, ey = err(x, y)
            h = 1e-7 * np.maximum(1.0, np.hypot(x, y))
            ax = (np.array(fisheye_radtan_distort(k, x + h, y, 1.0)) - np.array(fisheye_radtan_distort(k, x - h, y, 1.0))) / (2.0 * h)
            ay = (np.array(fisheye_radtan_distort(k, x, y + h, 1.0)) - np.array(fisheye_radtan_distort(k, x, y - h, 1.0))) / (2.0 * h)
            det = ax[0] * ay[1] - ay[0] * ax[1]
            sx, sy = -(ay[1] * ex - ay[0] * ey) / det, -(-ax[1] * ex + ax[0] * ey) / det
            t = np.ones_like(x)
            for _ in range(40):
                bad = ~(err(x + t * sx, y + t * sy)[0] <= e)
                if not bad.any():
                    break
                t = np.where(bad, 0.5 * t, t)
            moved = err(x + t * sx, y + t * sy)[0] <= e
            x, y = np.where(moved, x + t * sx, x), np.where(moved, y + t * sy, y)
        fx, fy = fisheye_radtan_distort(k, x, y, 1.0)
        ok = (np.hypot(fx - dx, fy - dy) <= 1e-12 * np.maximum(1.0, np.hypot(dx, dy))) & (np.arctan(np.hypot(x, y)) < thmax)
    return np.stack([x, y], axis=-1), ok


def project(model: int, intr, pts):
    """pts: (..., 3) camera-frame points -> (uv (..., 2), valid (...,))."""
    k = np.asarray(intr, dtype=np.float64)
    p = np.asarray(pts, dtype=np.float64)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    valid = np.ones(x.shape, dtype=bool)
    if model == PINHOLE:
        xn, yn = x / z, y / z
        r2 = xn * xn + yn * yn
        d = 1.0 + r2 * (k[5] + k[6] * r2)
        return _affine_skew(k, xn * d, yn * d), valid
    if model == PINHOLE_RADIAL_TANGENTIAL:
        xn, yn = x / z, y / z
        r2 = xn * xn + yn * yn
        d = 1.0 + r2 * (k[5] + r2 * (k[6] + r2 * k[7]))
        dx = xn * d + 2.0 * k[8] * xn * yn + k[9] * (r2 + 2.0 * xn * xn)
        dy = yn * d + 2.0 * k[9] * xn * yn + k[8] * (r2 + 2.0 * yn * yn)
        return _affine_skew(k, dx, dy), valid
    if model == FISHEYE:
        r2 = x * x + y * y
        r = np.sqrt(np.maximum(r2, 1e-300))
        th = np.arctan2(r, np.abs(z))
        th2 = th * th
        thd = th * (1.0 + th2 * (k[5] + th2 * (k[6] + th2 * (k[7] + th2 * k[8]))))
        sgn = np.where(z < 0, -1.0, 1.0)
        dx = np.where(r2 < 1e-8, x, sgn * thd * x / r)
        dy = np.where(r2 < 1e-8, y, sgn * thd * y / r)
        return _affine_skew(k, dx, dy), valid
    if model == FOV:
        xn, yn = x / z, y / z
        r2 = xn * xn + yn * yn
        om = k[4]
        r = np.sqrt(np.maximum(r2, 1e-300))
        if om * om < 1e-10:
            s = np.ones_like(r)
        else:
            s = np.where(r2 < 1e-10, 2.0 * np.tan(0.5 * om) / om, np.arctan(2.0 * r * np.tan(0.5 * om)) / (om * r))
        return np.stack([k[0] * s * xn + k[2], k[0] * k[1] * s * yn + k[3]], axis=-1), valid
    if model == DIVISION_UNDISTORTION:
        xu, yu = k[0] * x / z, k[0] * k[1] * y / z
        r2 = xu * xu + yu * yu
        den = 2.0 * k[4] * r2
        inner = 1.0 - 4.0 * k[4] * r2
        ident = (np.abs(den) < 1e-15) | (inner < 0.0)
        s = np.where(ident, 1.0, (1.0 - np.sqrt(np.maximum(inner, 0.0))) / np.where(ident, 1.0, den))
        return np.stack([xu * s + k[2], yu * s + k[3]], axis=-1), valid
    if model == DOUBLE_SPHERE:
        xi, al = k[5], k[6]
        r2 = x * x + y * y
        d1 = np.sqrt(r2 + z * z)
        w1 = _unified_w(al)
        w2 = (w1 + xi) / np.sqrt(2.0 * w1 * xi + xi * xi + 1.0)
        valid = z > -w2 * d1
        kk = xi * d1 + z
        d2 = np.sqrt(r2 + kk * kk)
        nrm = al * d2 + (1.0 - al) * kk
        return _affine_skew(k, x / nrm, y / nrm), valid
    if model == EXTENDED_UNIFIED:
        al, be = k[5], k[6]
        r2 = x * x + y * y
        rho = np.sqrt(be * r2 + z * z)
        nrm = al * rho + (1.0 - al) * z
        valid = z > -_unified_w(al) * rho
        return _affine_skew(k, x / nrm, y / nrm), valid
    if model == OMNI_RADIAL_TANGENTIAL:
        # unit sphere, then a pinhole at distance xi behind its centre; Kalibr's RadialTangentialDistortion without k3
        xi, k1, k2, t1, t2 = k[5], k[6], k[7], k[8], k[9]
        d = np.sqrt(x * x + y * y + z * z)
        valid = z > -(xi if xi <= 1.0 else 1.0 / xi) * d
        n = z + xi * d
        mx, my = x / n, y / n
        r2 = mx * mx + my * my
        radial = 1.0 + k1 * r2 + k2 * r2 * r2
        dx = mx * radial + 2.0 * t1 * mx * my + t2 * (r2 + 2.0 * mx * mx)
        dy = my * radial + 2.0 * t2 * mx * my + t1 * (r2 + 2.0 * my * my)
        return _affine_skew(k, dx, dy), valid
    if model == SCARAMUZZA:
        # OCamCalib's world2cam with the exact root: the sensor point s (x, y), then the stretch [[1, e], [d, c]] and the centre
        s, valid = scaramuzza_scale(k, np.hypot(x, y), z)
        up, vp = s * x, s * y
        return np.stack([up + k[2] * vp + k[3], k[8] * up + k[1] * vp + k[4]], axis=-1), valid
    if model == PINHOLE_RATIONAL:
        # OpenCV's projectPoints with CALIB_RATIONAL_MODEL (t1, t2 = p1, p2), valid iff z > 0 and s < s_max (which implies M(s) > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            xn, yn = x / z, y / z
            s = xn * xn + yn * yn
            dx, dy = rational_distort(k, xn, yn)
            valid = (z > 0.0) & (s < rational_s_max(k)) & (1.0 + s * (k[10] + s * (k[11] + s * k[12])) > 0.0)
        return _affine_skew(k, dx, dy), valid
    if model == FISHEYE_RADIAL_TANGENTIAL:
        # Kannala-Brandt with k1..k6, then the tangential terms (t1, t2 = OpenCV's p1, p2); valid iff z > 0 and theta < theta_max
        with np.errstate(divide="ignore", invalid="ignore"):
            dx, dy = fisheye_radtan_distort(k, x, y, z)
            valid = (z > 0.0) & (np.arctan2(np.hypot(x, y), z) < fisheye_radtan_theta_max(k))
        return _affine_skew(k, dx, dy), valid
    raise ValueError(f"unknown camera model {model}")
