"""Allan variance on the GPU (icc_allan_variance): factors, sigma^2 and tau of all six channels against the CPU oracle's sequential
calcVariance (always) and against the reference's own compiled code (oracle/_ref/allan_ref, when build() made it) at the small size,
at edge sizes and, for one accelerometer and one gyroscope channel, at full size; the six fits against the CPU oracle's fit of the
same curves; and the drop-in tool end to end."""
import ctypes
import json
import os
import subprocess
import time

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import calibrator, io_formats
from openimucameracalibrator_b200 import synthetic as syn
from allan_support import host_factors, oracle_factors, oracle_lib, oracle_variance, pushed, reference_curves

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")

pytestmark = pytest.mark.gpu


def oracle_curves(t, accel, gyro, channels=range(6), n_clusters=10000):
    """The oracle's sequential calcVariance of each channel's pushed values -> {channel: (factors, tau, sigma2)}."""
    out = {}
    for c in channels:
        tau, s2 = oracle_variance(t, pushed(dict(accel=accel, gyro=gyro), c), n_clusters)
        out[c] = (oracle_factors(len(t), n_clusters), tau, s2)
    return out


def edge_logs():
    """n/2 a power of two and its neighbours, including sizes whose last factor exceeds n/2 (the reference's 0/0 and -0)."""
    rng = np.random.default_rng(12)
    sizes = [n for n in (2 ** k for k in range(3, 17)) if host_factors(n, 10000)[-1] > n // 2][:3] + [3, 4, 1000, 16383, 16384, 16385]
    for n in sizes:
        yield n, np.cumsum(rng.uniform(0.004, 0.006, n)), rng.standard_normal((n, 3)) + 9.0, rng.standard_normal((n, 3)) * 0.01


def assert_curves_match(g, ref, channels):
    for c in channels:
        cv = g.allan_curves(c)
        fac, tau, s2 = ref[c]
        assert np.array_equal(cv["factors"], fac), c
        assert np.max(np.abs(cv["tau"] - tau) / np.abs(tau)) <= 1e-9, c
        np.testing.assert_array_equal(np.isnan(cv["sigma2"]), np.isnan(s2))
        np.testing.assert_array_equal(np.signbit(cv["sigma2"]), np.signbit(s2))
        ok = np.isfinite(s2) & (s2 != 0)
        err = np.max(np.abs(cv["sigma2"][ok] - s2[ok]) / np.abs(s2[ok]))
        assert err <= 1e-9, (c, err)


def test_gpu_variance_small_matches_oracle(gpu_factory):
    d = syn.allan_small()
    g = gpu_factory()
    g.allan_variance(d["t_s"], d["accel"], d["gyro"])
    assert_curves_match(g, oracle_curves(d["t_s"], d["accel"], d["gyro"]), range(6))


def test_gpu_variance_edge_sizes_match_oracle(gpu_factory):
    g = gpu_factory()
    for n, t, a, w in edge_logs():
        g.allan_variance(t, a, w)
        want = oracle_curves(t, a, w)
        assert_curves_match(g, want, range(6))
        if host_factors(n, 10000)[-1] > n // 2:   # the 0/0 or -0 point is there
            assert np.isnan(want[0][2][-1]) or np.signbit(want[0][2][-1]), n


def test_gpu_variance_many_factor_groups_match_oracle(gpu_factory):
    """200 000 clusters on 80 000 samples: 29 483 factors in 1 843 groups, more than one launch row holds, so CTAs take several
    groups in turn (the path that keeps any n_clusters within the grid limits)."""
    d = syn.make_allan_log(200.0, 400.0, 9)
    g = gpu_factory()
    g.allan_variance(d["t_s"], d["accel"], d["gyro"], n_clusters=200000)
    assert_curves_match(g, oracle_curves(d["t_s"], d["accel"], d["gyro"], n_clusters=200000), range(6))


def test_gpu_variance_small_matches_reference(gpu_factory, tmp_path):
    d = syn.allan_small()
    g = gpu_factory()
    g.allan_variance(d["t_s"], d["accel"], d["gyro"])
    assert_curves_match(g, reference_curves(tmp_path, d["t_s"], d["accel"], d["gyro"]), range(6))


def test_gpu_variance_edge_sizes_match_reference(gpu_factory, tmp_path):
    g = gpu_factory()
    for n, t, a, w in edge_logs():
        g.allan_variance(t, a, w)
        assert_curves_match(g, reference_curves(tmp_path, t, a, w), range(6))


def oracle_fit(c, freq, cv, mean_raw):
    f = oracle_lib().icca_fit_channel
    f.restype = None
    f.argtypes = [ctypes.c_int, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p,
                  ctypes.POINTER(capi.AllanNoise), ctypes.POINTER(capi.AllanSummary)]
    tau, s2 = np.ascontiguousarray(cv["tau"]), np.ascontiguousarray(cv["sigma2"])
    p, z, s = np.zeros(5), capi.AllanNoise(), capi.AllanSummary()
    f(c, freq, tau.size, tau.ctypes.data, s2.ctypes.data, mean_raw, p.ctypes.data, ctypes.byref(z), ctypes.byref(s))
    return p, z.as_dict(), s.as_dict()


@pytest.mark.parametrize("seed", [5, 8])
def test_gpu_fits_match_oracle(gpu_factory, seed):
    """Same points, initial values, iteration counts and terminations as the oracle's fit of the same curves.  The five-parameter
    fit is ill-conditioned and often ends at the 50-iteration limit, so the last-bit differences of the block-reduced normal
    equations (and the kernel's model decrease and Cauchy factor, formed from J^T J where the oracle uses the Jacobian rows) move the
parameters by up to about 1e-3 relative; final costs agree to 1e-6, the parameter-derived quantities to 1e-3."""
    d = syn.make_allan_log(200.0, 1200.0, seed)
    api = gpu_factory()
    r = api.allan_variance(d["t_s"], d["accel"], d["gyro"])
    for c in range(6):
        sg, zg = r["summary"][c], r["noise"][c]
        mean_raw = float(np.mean(pushed(d, c)))
        p, zo, so = oracle_fit(c, sg["freq"], api.allan_curves(c), mean_raw)
        assert sg["n_fit_points"] == so["n_fit_points"]
        assert sg["init_coeffs"] == so["init_coeffs"], c
        assert (sg["iterations"], sg["termination"], sg["successful_steps"]) == (so["iterations"], so["termination"], so["successful_steps"]), c
        assert abs(sg["initial_cost"] - so["initial_cost"]) <= 1e-12 * so["initial_cost"], c
        assert abs(sg["final_cost"] - so["final_cost"]) <= 1e-6 * so["final_cost"], (c, sg["final_cost"], so["final_cost"])
        assert abs(zg["mean"] - zo["mean"]) <= 1e-9 * abs(zo["mean"]), c
        for k in ("bias_instability", "white_noise", "white_noise_n", "bias_b"):
            assert abs(zg[k] - zo[k]) <= 1e-3 * abs(zo[k]), (c, k, zg[k], zo[k])


def test_gpu_full_size(gpu_factory, tmp_path):
    """2 h at 400 Hz (2.88 M samples): wall time of the whole call (incl. transfers); sigma^2 of acc_z (gravity) and gyr_x against
    the oracle's sequential calcVariance and, when available, the reference's own code (each about 15 s of CPU per channel)."""
    d = syn.allan_full_size()
    g = gpu_factory()
    g.allan_variance(d["t_s"], d["accel"], d["gyro"])
    times = []
    for _ in range(3):
        t0 = time.perf_counter(); r = g.allan_variance(d["t_s"], d["accel"], d["gyro"]); times.append(time.perf_counter() - t0)
    t1 = time.perf_counter(); want = oracle_curves(d["t_s"], d["accel"], d["gyro"], (2, 3)); tora = time.perf_counter() - t1
    assert_curves_match(g, want, (2, 3))
    s = r["summary"]
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = "?"
    print(f"\n[allan] n={s[0]['n_samples']} F={s[0]['n_factors']}: icc_allan_variance {min(times) * 1e3:.1f} ms wall (min of 3; "
          f"{[round(x * 1e3, 1) for x in times]} ms; internal {s[0]['seconds_total'] * 1e3:.1f} ms, {s[0]['gpu_launches']} launches) on {smi}; "
          f"sequential calcVariance of 2 channels on this host's CPU {tora:.1f} s; fit iterations {[x['iterations'] for x in s]}")
    if os.path.exists(os.path.join(ROOT, "oracle", "_ref", "allan_ref")):
        assert_curves_match(g, reference_curves(tmp_path, d["t_s"], d["accel"], d["gyro"], 10000, "23"), (2, 3))


def _write_telemetry(path, t_s, acc, gyr):
    t_ns = np.round(np.asarray(t_s) * 1e9)
    with open(path, "w") as f:
        json.dump({"timestamps_ns": t_ns.tolist(), "accelerometer": np.asarray(acc).tolist(), "gyroscope": np.asarray(gyr).tolist()}, f)
    return t_ns * 1e-9


def test_gpu_cli_end_to_end(gpu_factory, tmp_path):
    d = syn.allan_small()
    tel, out = str(tmp_path / "telemetry.json"), str(tmp_path / "allan.json")
    t = _write_telemetry(tel, d["t_s"], d["accel"], d["gyro"])
    p = subprocess.run([os.path.join(BIN, "fit_allan_variance"), f"--telemetry_json={tel}", f"--output_json={out}", "--verbose"], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    lines = p.stdout.splitlines()
    for label in ("Loading datastructes", "gyr_x  numData 240000", "gyr_x  freq ", "Gyro X ", " Bias Instability ", " White Noise ", "  bias ", "acc z ", "acc_z  period "):
        assert any(l.startswith(label) for l in lines), label
    assert sum(" rad/s, at " in l for l in lines) == 3 and sum(l.endswith(" m/s^2") for l in lines) == 6
    assert not any("Too few number" in l or "Too short time" in l for l in lines)
    c_lines = [l[2:] for l in lines if l.startswith("C ")]
    assert len(c_lines) == 6
    for body in c_lines:   # Eigen's row print: five coefficients right-aligned to the widest, one space apart
        w = (len(body) - 4) // 5
        assert len(body) == 5 * w + 4 and max(len(v) for v in body.split()) == w, body
        cells = [body[i * (w + 1):i * (w + 1) + w] for i in range(5)]
        assert all(x.strip() and x.rstrip() == x for x in cells), body   # right-aligned, nothing empty
        [float(x) for x in cells]
    api = gpu_factory()
    r = api.allan_variance(t, d["accel"], d["gyro"])
    want = io_formats.allan_variance_document(r, [api.allan_curves(c) for c in range(6)])
    assert json.load(open(out)) == json.loads(json.dumps(want))
    # the reference's warnings on a short log
    short = syn.make_allan_log(100.0, 60.0, 2)
    _write_telemetry(tel, short["t_s"], short["accel"], short["gyro"])
    q = subprocess.run([os.path.join(BIN, "fit_allan_variance"), f"--telemetry_json={tel}"], capture_output=True, text=True)
    assert q.returncode == 0, q.stderr
    assert "gyr_x  Too few number" in q.stdout and "acc_x  Too short time!!!!" in q.stdout


def test_gpu_python_mirror(gpu_factory):
    d = syn.make_allan_log(200.0, 600.0, 3)
    f = calibrator.AllanVarianceFitter(d["t_s"], d["accel"], d["gyro"], 10000)
    assert f.RunFit()
    r = gpu_factory().allan_variance(d["t_s"], d["accel"], d["gyro"])
    assert np.array_equal(f.params, r["params"]) and f.noise == r["noise"]
    assert f.curves(4)["sigma2"].size == r["summary"][4]["n_factors"]
