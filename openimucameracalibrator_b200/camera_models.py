"""NumPy camera projections used by the synthetic-data generator (host-side, FP64).

Third, independent statement of the Theia camera-model equations that the reference dispatches at
include/OpenCameraCalibrator/basalt_spline/ceres_calib_split_residuals.h:366-389 (the device statement lives in
csrc/icc_camera.cuh, the autodiff statement in oracle/oracle_math.hpp).  Model ids are theia::CameraIntrinsicsModelType
values; JSON names follow src/io/read_camera_calibration.cc:59-116.
"""
from __future__ import annotations

import numpy as np

PINHOLE, PINHOLE_RADIAL_TANGENTIAL, FISHEYE, FOV, DIVISION_UNDISTORTION, DOUBLE_SPHERE, EXTENDED_UNIFIED = range(7)
OMNI_RADIAL_TANGENTIAL = 7   # extension without a Theia counterpart: Kalibr's omni-radtan

MODEL_NAMES = {
    PINHOLE: "PINHOLE",
    PINHOLE_RADIAL_TANGENTIAL: "PINHOLE_RADIAL_TANGENTIAL",
    FISHEYE: "FISHEYE",
    FOV: "FOV",
    DIVISION_UNDISTORTION: "DIVISION_UNDISTORTION",
    DOUBLE_SPHERE: "DOUBLE_SPHERE",
    EXTENDED_UNIFIED: "EXTENDED_UNIFIED",
    OMNI_RADIAL_TANGENTIAL: "OMNI_RADIAL_TANGENTIAL",
}
MODEL_IDS = {v: k for k, v in MODEL_NAMES.items()}
NUM_PARAMS = {PINHOLE: 7, PINHOLE_RADIAL_TANGENTIAL: 10, FISHEYE: 9, FOV: 5, DIVISION_UNDISTORTION: 5,
              DOUBLE_SPHERE: 7, EXTENDED_UNIFIED: 7, OMNI_RADIAL_TANGENTIAL: 10}


def _affine_skew(k, dx, dy):
    return np.stack([k[0] * dx + k[2] * dy + k[3], k[0] * k[1] * dy + k[4]], axis=-1)


def _unified_w(alpha):
    return (1.0 - alpha) / alpha if alpha > 0.5 else alpha / (1.0 - alpha)


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
    raise ValueError(f"unknown camera model {model}")
