"""Shared pieces of the bias random-walk tests: the oracle with the bias-spline spacing and the prior (tests/bias_walk/bias_walk_oracle.cpp),
the product's prior rows compiled for the CPU (tests/bias_walk/bias_walk_host_math.cu), a NumPy statement of the prior by dense quadrature,
and a camera-IMU sequence whose biases drift: a random walk of known density plus a warm-up exponential."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
DP = ctypes.POINTER(ctypes.c_double)
_LIB, _HM = None, None


def new_bias_walk_oracle() -> capi.CApi:
    """the CPU oracle with every camera model, the tangent residual, the bias-spline spacing and the random-walk prior"""
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_bias_walk_oracle_"), "libicc_bias_walk_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(HERE, "bias_walk", "bias_walk_oracle.cpp")])
        _LIB = ctypes.CDLL(out)
    return capi.CApi(_LIB, "icco_", 0)


def host_math():
    """the product's icc_bias_prior.cuh compiled for the CPU"""
    global _HM
    if _HM is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_bias_walk_hm_"), "libbias_walk_hm.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", out,
                               os.path.join(HERE, "bias_walk", "bias_walk_host_math.cu")])
        _HM = ctypes.CDLL(out)
        _HM.bw_prior_rows.restype = ctypes.c_int
        _HM.bw_prior_rows.argtypes = [ctypes.c_int, DP, ctypes.c_double, DP, DP]
    return _HM


def host_rows(knots, dt_s, q):
    """the product's prior rows of one sensor's knots (n, 3), in the residual order of icc_evaluate"""
    k = np.ascontiguousarray(knots, dtype=np.float64); qq = np.ascontiguousarray(np.broadcast_to(q, (3,)), dtype=np.float64)
    out = np.zeros(6 * (k.shape[0] - 2))
    assert host_math().bw_prior_rows(k.shape[0], k.ctypes.data_as(DP), float(dt_s), qq.ctypes.data_as(DP), out.ctypes.data_as(DP)) == out.size
    return out


def prior_integral(knots, dt_s, q, nodes=12):
    """1/2 int |b'(t)|^2 / q^2 dt over all n - 2 segments of the spline, by `nodes`-point Gauss-Legendre per segment"""
    k = np.asarray(knots, dtype=np.float64); q = np.broadcast_to(np.asarray(q, dtype=np.float64), (3,))
    x, w = np.polynomial.legendre.leggauss(nodes)
    u, w = 0.5 * (x + 1.0), 0.5 * w
    dB = np.stack([-(1.0 - u), 1.0 - 2.0 * u, u], -1)                      # (nodes, 3)
    total = 0.0
    for s in range(k.shape[0] - 2):
        bdot = dB @ k[s:s + 3] / dt_s                                       # (nodes, 3 axes)
        total += 0.5 * dt_s * np.sum(w[:, None] * bdot ** 2 / q ** 2)
    return total


def prior_rows_of(api):
    """the prior rows of an evaluation (they follow the gyroscope rows)"""
    _, r, _, _ = api.evaluate(capi.FLAG_SPLINE | capi.FLAG_T_I_C, gradient=False)
    return r[sum(api.num_residuals()):]


def imu_segments(o):
    """per used IMU sample of the oracle: (s_so3, s_r3, s_acc_bias, s_gyr_bias)"""
    n = len(o.imu_used()[0])
    seg = np.full((n, 4), -1, dtype=np.int32)
    o._call("get_imu_segments", [ctypes.POINTER(ctypes.c_int32)], seg.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)))
    return seg


def cells_from_segments(seg):
    """maximal runs of samples with equal segment indices: rows (s_so3, s_r3, s_acc_bias, s_gyr_bias, i_begin, i_end)"""
    cells = []
    for i, s in enumerate(seg):
        if cells and tuple(cells[-1][:4]) == tuple(s):
            cells[-1][5] = i + 1
        else:
            cells.append([*map(int, s), i, i + 1])
    return np.array(cells, dtype=np.int32).reshape(-1, 6)


# ---- a sequence whose biases drift -------------------------------------------------------------------------------------------------------
# a walk that wanders on a scale of seconds (what 10 s knots cannot follow) and a slow warm-up of a few times the walk's own rate
DRIFT = dict(acc_q=2e-2, gyr_q=2e-3, acc_warm=(0.05, -0.04, 0.03), gyr_warm=(2e-3, -1.5e-3, 1e-3), tau_s=20.0)


def drifting_dataset(n_frames=1200, seed=31, drift=DRIFT, **kw):
    """The synthetic sequence of syn.make_dataset (its outputs untouched) with time-varying biases added to the IMU readings:
    b(t) = b0 + warm (1 - exp(-t / tau)) + a random walk of density q per axis (m/s^3/sqrt(Hz), rad/s^2/sqrt(Hz)).  The dataset gains
    "bias_truth": the true biases (acc, gyr) of every IMU sample at its camera-clock time t_cam, the spline's time axis."""
    cfg = syn.tiny_config(n_frames=n_frames, grid=(6, 5), imu_rate_hz=200.0, seed=seed, **kw)
    ds = syn.make_dataset(cfg)
    rng = np.random.default_rng(seed + 1000)
    t_cam = np.asarray(ds["imu_t"]) + ds["time_offset_imu_to_cam_s"]          # camera-clock time of every sample
    dt = np.diff(t_cam, prepend=t_cam[0])
    rel = t_cam - t_cam[0]
    out = dict(ds)
    truth = {}
    for key, read, b0 in (("acc", "accel", ds["acc_bias"]), ("gyr", "gyro", ds["gyr_bias"])):
        walk = np.cumsum(drift[key + "_q"] * np.sqrt(dt)[:, None] * rng.standard_normal((t_cam.size, 3)), axis=0)
        warm = np.asarray(drift[key + "_warm"])[None] * (1.0 - np.exp(-rel / drift["tau_s"]))[:, None]
        out[read] = np.asarray(ds[read]) + walk + warm
        truth[key] = np.asarray(b0)[None] + walk + warm
    out["bias_truth"] = dict(t_cam=t_cam, **truth)
    return out
