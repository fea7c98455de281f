"""Allan variance characterisation without a GPU: the factor set and the oracle's variance against the reference's own compiled
code, the oracle's fit against the synthetic truth, the dogleg step control of icc_trust_region.cuh against a short statement of
its rules, the JSON document, and the new C-ABI symbols' behaviour without a device."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import calibrator, io_formats
from openimucameracalibrator_b200 import synthetic as syn
from allan_support import host_factors, host_math_lib, new_allan_oracle, oracle_factors, oracle_variance, pushed, reference_curves

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")

FACTOR_SIZES = [3, 4, 5, 7, 100, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097, 9999, 16383, 16384, 16385, 32767, 32768, 32769]


@pytest.mark.parametrize("n_clusters", [2, 100, 10000])
def test_factor_set_equals_oracle_restatement(n_clusters):
    for n in FACTOR_SIZES + [65536, 131072, 131073, 262143, 262144, 2880000]:
        assert np.array_equal(host_factors(n, n_clusters), oracle_factors(n, n_clusters)), n


@pytest.mark.parametrize("n_clusters", [2, 100, 10000])
def test_factor_set_equals_reference(tmp_path, n_clusters):
    rng = np.random.default_rng(1)
    for n in FACTOR_SIZES:
        t = np.arange(n) * 0.005
        ref = reference_curves(tmp_path, t, rng.standard_normal((n, 3)), rng.standard_normal((n, 3)), n_clusters, "0")
        assert np.array_equal(host_factors(n, n_clusters), ref[0][0]), n


def test_factor_set_edge_exceeds_max_stride():
    """Where ceil of the last log-space value passes the largest power of two <= n/2, the last factor is maxStride + 1."""
    hits = [n for n in (2 ** k for k in range(2, 23)) if host_factors(n, 10000)[-1] > n // 2]
    assert hits, "no size with a factor above n/2 among the powers of two"


def test_oracle_variance_equals_reference(tmp_path):
    d = syn.make_allan_log(rate_hz=100.0, duration_s=300.0, seed=3)
    ref = reference_curves(tmp_path, d["t_s"], d["accel"], d["gyro"], 10000, "03")
    for c in (0, 3):
        tau, s2 = oracle_variance(d["t_s"], pushed(d, c))
        assert np.array_equal(tau, ref[c][1])
        assert np.max(np.abs(s2 - ref[c][2]) / np.abs(ref[c][2])) <= 1e-12, c


def test_oracle_variance_edge_sizes_equal_reference(tmp_path):
    """Sizes whose last factor makes n - 2m zero or negative: the reference's 0/0 and -0 are kept."""
    rng = np.random.default_rng(2)
    for n in [n for n in (2 ** k for k in range(2, 16)) if host_factors(n, 10000)[-1] > n // 2][:4]:
        t = np.arange(n) * 0.01
        a, g = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
        ref = reference_curves(tmp_path, t, a, g, 10000, "0")
        _, s2 = oracle_variance(t, a[:, 0])
        np.testing.assert_array_equal(np.signbit(s2), np.signbit(ref[0][2]))
        np.testing.assert_array_equal(np.isnan(s2), np.isnan(ref[0][2]))
        ok = np.isfinite(ref[0][2]) & (ref[0][2] != 0)
        assert np.max(np.abs(s2[ok] - ref[0][2][ok]) / np.abs(ref[0][2][ok])) <= 1e-12


def test_oracle_fit_recovers_synthetic_truth():
    """White noise to 5 % on every axis; the bias random walk, which a 30-minute log only starts to show, to the same order on
    average over the three axes of each sensor.  The model is even in each parameter, so magnitudes are compared."""
    d = syn.make_allan_log(rate_hz=100.0, duration_s=1800.0, seed=4)
    tr = d["truth"]
    r = new_allan_oracle().allan_variance(d["t_s"], d["accel"], d["gyro"])
    for sensor in (0, 1):
        scale = 1.0 if sensor == 0 else 57.3 * 3600
        white, walk = (tr["acc_white"], tr["acc_walk"]) if sensor == 0 else (tr["gyr_white"], tr["gyr_walk"])
        k_ratio = []
        for c in range(3 * sensor, 3 * sensor + 3):
            s = r["summary"][c]
            assert s["termination"] in (0, 1, 2, 3) and s["final_cost"] < s["initial_cost"], (c, s)
            assert abs(abs(r["params"][c][1]) / (white * scale) - 1.0) < 0.05, (c, r["params"][c])
            k_ratio.append(abs(r["params"][c][3]) / (walk / np.sqrt(3) * scale))
        assert 1 / 3 < np.mean(k_ratio) < 3, k_ratio


# ---- dogleg step control (icc_trust_region.cuh) against a statement of the rules --------------------------------------------------
def dogleg_rules(rows, cost0):
    st = dict(radius=1e4, mu=1e-8, step_norm=0.0, reuse=0, term=-1, it=0, succ=0, invalid=0, cost=cost0)
    out = []
    for valid, mc, sn, xn, cand, dl in rows:
        if st["term"] < 0 and st["it"] >= 50:
            st["term"] = 0
        if st["term"] < 0:
            st["step_norm"] = dl
            st["it"] += 1
            if not valid or not mc > 0:
                st["invalid"] += 1
                if st["invalid"] >= 5:
                    st["term"] = 4
                else:
                    st["mu"] *= 10; st["reuse"] = 0
            else:
                st["invalid"] = 0
                if sn <= 1e-8 * (xn + 1e-8):
                    st["term"] = 2
                else:
                    cand = cand if np.isfinite(cand) else 1.7976931348623157e308
                    change = st["cost"] - cand
                    rho = change / mc
                    if abs(change) <= 1e-6 * st["cost"]:
                        st["term"] = 1
                    elif not rho > 1e-3:
                        st["radius"] *= 0.5; st["reuse"] = 1
                        if st["radius"] < 1e-32:
                            st["term"] = 4
                    else:
                        st["succ"] += 1; st["cost"] = cand
                        if rho < 0.25:
                            st["radius"] *= 0.5
                        if rho > 0.75:
                            st["radius"] = max(st["radius"], 3 * dl)
                        if st["radius"] < 1e-32:
                            st["term"] = 4
                        st["mu"] = max(1e-8, 2 * st["mu"] / 10); st["reuse"] = 0
        out.append([st["radius"], st["mu"], st["step_norm"], st["reuse"], st["term"], st["it"], st["succ"], st["invalid"], st["cost"]])
    return np.array(out, dtype=float)


def run_script(rows, cost0):
    rows = np.ascontiguousarray(rows, dtype=float)
    out = np.zeros((len(rows), 9))
    f = host_math_lib().ah_dogleg_script
    f.restype = None; f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p]
    f(len(rows), rows.ctypes.data, float(cost0), out.ctypes.data)
    return out


def test_dogleg_scripted_transitions():
    cost0 = 10.0
    rows = [
        (1, 2.0, 1.0, 1.0, 9.0, 50.0),      # rho 0.5: accepted, radius kept, mu stays at its minimum
        (1, 1.0, 1.0, 1.0, 8.05, 5e3),      # rho 0.95: radius max(radius, 3 |step|) = 1.5e4
        (1, 1.0, 1.0, 1.0, 7.95, 1.0),      # rho 0.1: accepted, radius halved
        (1, 1.0, 1.0, 1.0, 9.0, 1.0),       # cost increase: rejected, radius halved, vectors reused
        (0, 0.0, 1.0, 1.0, 0.0, 1.0),       # solve failed: invalid, mu x 10, no reuse
        (1, -1.0, 1.0, 1.0, 0.0, 1.0),      # no model decrease: invalid, mu x 10
        (1, 1.0, 1.0, 1.0, 7.0, 1.0),       # accepted: mu / 5
        (1, 1.0, 1.0, 1.0, 7.0 - 1e-7, 1.0),  # function tolerance
    ]
    np.testing.assert_array_equal(run_script(rows, cost0), dogleg_rules(rows, cost0))
    five_invalid = [(0, 0.0, 1.0, 1.0, 0.0, 1.0)] * 6
    got = run_script(five_invalid, cost0)
    np.testing.assert_array_equal(got, dogleg_rules(five_invalid, cost0))
    assert got[4, 4] == 4 and got[4, 1] == pytest.approx(1e-4)
    tiny = [(1, 1.0, 1e-12, 1.0, 5.0, 1.0)]    # parameter tolerance: no candidate considered
    assert run_script(tiny, cost0)[0, 4] == 2
    many_rejects = [(1, 1.0, 1.0, 1.0, 11.0, 1.0)] * 60   # 50 iterations then max_iterations
    np.testing.assert_array_equal(run_script(many_rejects, cost0), dogleg_rules(many_rejects, cost0))


def test_dogleg_random_transitions():
    rng = np.random.default_rng(9)
    for _ in range(200):
        k = int(rng.integers(1, 60))
        cost0 = float(rng.uniform(1, 100))
        rows = []
        for _ in range(k):
            kind = rng.integers(0, 6)
            mc = float(rng.uniform(0.01, 2.0)) if kind else float(-rng.uniform(0, 1))
            rows.append((float(kind != 1), mc, float(10 ** rng.uniform(-12, 1)), float(rng.uniform(0, 2)),
                         float(cost0 * rng.uniform(0.5, 1.2)), float(10 ** rng.uniform(-2, 5))))
        np.testing.assert_array_equal(run_script(rows, cost0), dogleg_rules(rows, cost0))


def dogleg_step_rules(g, gn, D, alpha, radius):
    gnorm, nnorm = np.linalg.norm(g), np.linalg.norm(gn)
    if nnorm <= radius:
        return gn / D, nnorm
    if gnorm * alpha >= radius:
        return -(radius / gnorm) * g / D, radius
    a, b = -alpha * g, gn
    beta = np.roots([np.dot(b - a, b - a), 2 * np.dot(a, b - a), np.dot(a, a) - radius ** 2]).real.max()
    s = a + beta * (b - a)
    return s / D, np.linalg.norm(s)


def test_dogleg_step_cases():
    rng = np.random.default_rng(3)
    f = host_math_lib().ah_dogleg_step
    f.restype = ctypes.c_double; f.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_double, ctypes.c_double, ctypes.c_void_p]
    cases = set()
    for _ in range(300):
        g, gn, D = rng.standard_normal(5), rng.standard_normal(5) * 3, rng.uniform(0.5, 2, 5)
        alpha, radius = float(rng.uniform(0.1, 1)), float(10 ** rng.uniform(-1, 1))
        step = np.zeros(5)
        norm = f(g.ctypes.data, gn.ctypes.data, D.ctypes.data, alpha, radius, step.ctypes.data)
        want, wn = dogleg_step_rules(g, gn, D, alpha, radius)
        np.testing.assert_allclose(step, want, rtol=1e-9, atol=1e-12)
        assert norm == pytest.approx(wn, rel=1e-12)
        cases.add(0 if np.linalg.norm(gn) <= radius else (1 if np.linalg.norm(g) * alpha >= radius else 2))
    assert cases == {0, 1, 2}


# ---- documents, CLI and C-ABI without a device -------------------------------------------------------------------------------------
def test_allan_json_document(tmp_path):
    F = 4
    res = dict(params=np.arange(30.0).reshape(6, 5),
               noise=[dict(mean=1.0, bias_instability=2.0, bias_instability_tau=3.0, bias_b=4.0, white_noise_n=5.0, white_noise=6.0)] * 6,
               summary=[dict(n_samples=100, freq=200.0, period=0.005, n_fit_points=F, iterations=7, termination=1, initial_cost=2.0, final_cost=1.0)] * 6)
    curves = [dict(factors=np.arange(1, F + 1), tau=np.arange(1, F + 1) * 0.005, sigma2=np.ones(F), fit_deviation=np.ones(F))] * 6
    p = str(tmp_path / "allan.json")
    io_formats.write_allan_variance_json(p, res, curves)
    doc = json.load(open(p))
    assert list(doc["channels"]) == list(capi.ALLAN_CHANNELS)
    ch = doc["channels"]["gyr_x"]
    assert ch["params"] == {"Q": 15.0, "N": 16.0, "B": 17.0, "K": 18.0, "R": 19.0}
    assert ch["tau"] == [0.005, 0.01, 0.015, 0.02] and ch["fit"]["iterations"] == 7.0
    assert set(ch) == {"factors", "tau", "sigma2", "fit_deviation", "params", "noise", "fit"}
    assert set(doc) == {"n_samples", "freq", "period", "channels"}


def _write_telemetry(path, t_s, acc, gyr):
    with open(path, "w") as f:
        json.dump({"timestamps_ns": np.round(np.asarray(t_s) * 1e9).tolist(), "accelerometer": np.asarray(acc).tolist(), "gyroscope": np.asarray(gyr).tolist()}, f)


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the no-device path is exercised on the CPU box")


def test_cli_without_device_fails_loudly(tmp_path):
    _no_gpu()
    d = syn.make_allan_log(rate_hz=50.0, duration_s=20.0)
    tel = str(tmp_path / "telemetry.json")
    _write_telemetry(tel, d["t_s"], d["accel"], d["gyro"])
    p = subprocess.run([os.path.join(BIN, "fit_allan_variance"), f"--telemetry_json={tel}"], capture_output=True, text=True)
    assert p.returncode == 2 and "icc_create failed" in p.stderr
    q = subprocess.run([os.path.join(BIN, "fit_allan_variance"), "--telemetry_json=/nonexistent.json"], capture_output=True, text=True)
    assert q.returncode == 1 and "Could not read" in q.stderr


def test_capi_allan_without_device():
    _no_gpu()
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    t = np.arange(10) * 0.01
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h.allan_variance(t, np.ones((10, 3)), np.ones((10, 3)))
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):   # the reference divides by zero here
        h.allan_variance(t[:2], np.ones((2, 3)), np.ones((2, 3)))
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
        h.allan_variance(t, np.ones((10, 3)), np.ones((10, 3)), n_clusters=1)
    assert h.allan_curves(0)["factors"].size == 0
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
        h.allan_curves(6)
