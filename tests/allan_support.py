"""Loaders of the Allan variance test libraries (tests/allan/): the CPU oracle (g++), the kernels' host math compiled for the CPU
(nvcc, host code only), both built once per process into a temporary directory, and the reference's own Allan variance code that
build() compiles into oracle/_ref/allan_ref when a reference checkout is available."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from openimucameracalibrator_b200._capi import CApi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "allan")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "allan_ref")
_BUILD = None
_LIBS = {}


def _build_dir():
    global _BUILD
    if _BUILD is None:
        _BUILD = tempfile.mkdtemp(prefix="icc_allan_")
    return _BUILD


def _lib(name, cmd):
    if name not in _LIBS:
        out = os.path.join(_build_dir(), f"lib{name}.so")
        subprocess.check_call(cmd(out))
        _LIBS[name] = ctypes.CDLL(out)
    return _LIBS[name]


def oracle_lib():
    return _lib("allan_oracle", lambda out: ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, os.path.join(SRC, "allan_oracle.cpp")])


def host_math_lib():
    return _lib("allan_host_math", lambda out: ["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                                                 "-Wno-deprecated-gpu-targets", "-o", out, os.path.join(SRC, "allan_host_math.cu")])


def new_allan_oracle() -> CApi:
    return CApi(oracle_lib(), "icca_", 0)


def _i32(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def oracle_factors(n, n_clusters):
    f = oracle_lib().icca_factors
    f.restype = ctypes.c_int; f.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int32), ctypes.c_int]
    buf = np.zeros(n_clusters, dtype=np.int32)
    k = f(n, n_clusters, _i32(buf), n_clusters)
    return buf[:k].astype(np.int64)


def host_factors(n, n_clusters):
    f = host_math_lib().ah_factors
    f.restype = ctypes.c_int; f.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int32), ctypes.c_int]
    buf = np.zeros(n_clusters, dtype=np.int32)
    k = f(n, n_clusters, _i32(buf), n_clusters)
    return buf[:k].astype(np.int64)


def oracle_variance(t, x, n_clusters=10000):
    """The oracle's sequential calcVariance of one channel's pushed values -> (tau, sigma2)."""
    t = np.ascontiguousarray(t, dtype=np.float64); x = np.ascontiguousarray(x, dtype=np.float64)
    F = oracle_factors(t.size, n_clusters).size
    tau, s2 = np.zeros(F), np.zeros(F)
    f = oracle_lib().icca_variance
    f.restype = None; f.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double), ctypes.c_int,
                                    ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]
    f(t.size, _dp(t), _dp(x), n_clusters, _dp(tau), _dp(s2))
    return tau, s2


def pushed(d, c):
    """Channel c's values as AllanVarianceFitter pushes them (gyroscope rad/s -> deg/h as (x * 57.3) * 3600)."""
    return d["accel"][:, c] if c < 3 else d["gyro"][:, c - 3] * 57.3 * 3600


def need_reference():
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/allan_ref absent: build() compiles it only when ICC_REFERENCE_ROOT names a reference checkout")
    return REF_BIN


def reference_curves(tmpdir, t, accel, gyro, n_clusters=10000, channels="012345"):
    """Runs the reference's own AllanAcc / AllanGyr -> {channel: (factors, tau, sigma2)}."""
    exe = need_reference()
    t = np.ascontiguousarray(t, dtype=np.float64)
    inp, out = os.path.join(str(tmpdir), "allan_in.bin"), os.path.join(str(tmpdir), "allan_out.bin")
    with open(inp, "wb") as f:
        f.write(np.int64(t.size).tobytes()); f.write(t.tobytes())
        f.write(np.ascontiguousarray(accel, dtype=np.float64).tobytes()); f.write(np.ascontiguousarray(gyro, dtype=np.float64).tobytes())
    subprocess.run([exe, inp, out, str(n_clusters), channels], check=True, stdout=subprocess.DEVNULL)
    buf = open(out, "rb").read()
    res, k = {}, 0
    while k < len(buf):
        c, F = np.frombuffer(buf, np.int32, 2, k); k += 8
        fac = np.frombuffer(buf, np.int32, F, k).astype(np.int64); k += 4 * F
        tau = np.frombuffer(buf, np.float64, F, k); k += 8 * F
        s2 = np.frombuffer(buf, np.float64, F, k); k += 8 * F
        res[int(c)] = (fac, tau, s2)
    return res
