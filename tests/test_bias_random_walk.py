"""Bias-spline spacing and the random-walk prior on the bias splines, without a GPU: the product's prior rows (icc_bias_prior.cuh compiled
for the CPU) and the oracle's against a dense quadrature of the Wiener-process likelihood, the assembly of a host-only handle against the
oracle's, the setters' argument checks, the Allan-fit conversion, sharding and the CLI's flag rules."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from bias_walk_support import cells_from_segments, host_rows, imu_segments, new_bias_walk_oracle, prior_integral, prior_rows_of
from openimucameracalibrator_b200 import _capi as capi, calibrator, io_formats, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
F_BIAS = capi.FLAG_SPLINE | capi.FLAG_T_I_C | capi.FLAG_IMU_BIASES


def _ds(n_frames=24, **kw):
    return syn.make_dataset(syn.tiny_config(n_frames=n_frames, **kw))


def _host(ds, spacing=None, walk=None, shard=None):
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    if spacing is not None:
        h.set_bias_splines(*spacing)
    if walk is not None:
        h.set_bias_random_walk(*walk)
    capi.load_dataset(h, ds, known_gravity=False, shard=shard)
    return h


def _oracle(ds, spacing=None, walk=None, shard=None):
    o = new_bias_walk_oracle()
    if spacing is not None:
        o.set_bias_splines(*spacing)
    if walk is not None:
        o.set_bias_random_walk(*walk)
    capi.load_dataset(o, ds, shard=shard)
    return o


# ---- the rows ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [0.37, 2.0, 10.0])
def test_host_rows_are_the_integral(dt):
    rng = np.random.default_rng(int(dt * 100))
    q = np.array([2e-3, 5e-3, 1e-3])
    for n in (3, 4, 17):
        k = rng.normal(0.0, 0.05, (n, 3))
        r = host_rows(k, dt, q)
        assert r.size == 6 * (n - 2)
        ref = prior_integral(k, dt, q)
        assert abs(0.5 * np.sum(r * r) - ref) <= 1e-12 * ref
        # Jacobian: constant, against central differences
        eps = 1e-6
        for i in range(n):
            for a in range(3):
                kp, km = k.copy(), k.copy(); kp[i, a] += eps; km[i, a] -= eps
                fd = (host_rows(kp, dt, q) - host_rows(km, dt, q)) / (2 * eps)
                s = np.arange(r.size).reshape(n - 2, 2, 3)
                want = np.zeros(r.size)
                for seg in range(max(0, i - 2), min(i, n - 3) + 1):
                    for g, u in enumerate((0.5 - 0.5 / np.sqrt(3), 0.5 + 0.5 / np.sqrt(3))):
                        want[s[seg, g, a]] = (-(1 - u), 1 - 2 * u, u)[i - seg] / (q[a] * np.sqrt(2 * dt))
                np.testing.assert_allclose(fd, want, rtol=1e-7, atol=1e-6 * np.abs(want).max())


def test_equal_knots_cost_nothing_and_a_ramp_costs_its_integral():
    k = np.tile([0.1, -0.2, 0.05], (9, 1))
    assert np.all(host_rows(k, 1.5, 1e-3) == 0.0)
    dt, n, a, q = 1.5, 9, np.array([1e-3, -2e-3, 5e-4]), np.array([2e-3, 1e-3, 4e-3])
    ramp = np.arange(n)[:, None] * dt * a[None] + 0.3
    r = host_rows(ramp, dt, q)
    T = (n - 2) * dt
    np.testing.assert_allclose(0.5 * np.sum(r * r), np.sum(a * a * T / (2 * q * q)), rtol=1e-12)


@pytest.mark.parametrize("dt", [0.25, 0.5, 10.0])
def test_oracle_rows_equal_the_product_rows_and_the_integral(dt):
    ds = _ds()
    q_a, q_g = np.array([2e-3, 3e-3, 1e-3]), np.array([1e-4, 2e-4, 3e-4])
    o = _oracle(ds, spacing=(dt, dt), walk=(q_a, q_g))
    rng = np.random.default_rng(3)
    so3, r3, ba, bg = o.get_knots()
    ba = ba + rng.normal(0, 0.02, ba.shape); bg = bg + rng.normal(0, 2e-3, bg.shape)
    o.set_knots(ba=ba, bg=bg)
    rows = prior_rows_of(o)
    assert rows.size == o.num_bias_prior_residuals() == 6 * (ba.shape[0] - 2) + 6 * (bg.shape[0] - 2)
    ha, hg = host_rows(ba, dt, q_a), host_rows(bg, dt, q_g)
    np.testing.assert_allclose(rows, np.concatenate([ha, hg]), rtol=1e-13, atol=1e-13 * np.abs(rows).max())
    want = prior_integral(ba, dt, q_a) + prior_integral(bg, dt, q_g)
    assert abs(0.5 * np.sum(rows * rows) - want) <= 1e-12 * want
    # the oracle's cost is the data's plus the prior's
    base = _oracle(ds, spacing=(dt, dt)); base.set_knots(ba=ba, bg=bg)
    c1, c0 = o.evaluate(F_BIAS, residuals=False, gradient=False)[0], base.evaluate(F_BIAS, residuals=False, gradient=False)[0]
    assert abs(c1 - c0 - want) <= 1e-9 * want


def test_oracle_prior_jacobian_against_central_differences():
    ds = _ds()
    o = _oracle(ds, spacing=(0.3, 0.3), walk=(2e-3, 2e-4))
    so3, r3, ba, bg = o.get_knots()
    flags = capi.FLAG_IMU_BIASES
    n = o.num_tangent(flags)
    J = np.zeros((sum(o.num_residuals()) + o.num_bias_prior_residuals(), n))
    o._call("jacobian_dense", [ctypes.c_int, ctypes.POINTER(ctypes.c_double)], flags, J.ctypes.data_as(ctypes.POINTER(ctypes.c_double)))
    Jp = J[sum(o.num_residuals()):]
    eps = 1e-6
    for col, (which, i, a) in enumerate([(w, i, a) for w, arr in (("ba", ba), ("bg", bg)) for i in range(arr.shape[0]) for a in range(3)]):
        arrs = {"ba": ba.copy(), "bg": bg.copy()}
        arrs[which][i, a] += eps; o.set_knots(ba=arrs["ba"], bg=arrs["bg"]); rp = prior_rows_of(o)
        arrs[which][i, a] -= 2 * eps; o.set_knots(ba=arrs["ba"], bg=arrs["bg"]); rm = prior_rows_of(o)
        np.testing.assert_allclose((rp - rm) / (2 * eps), Jp[:, col], rtol=1e-6, atol=1e-6 * np.abs(Jp).max())
    o.set_knots(ba=ba, bg=bg)


# ---- assembly on a host-only handle -------------------------------------------------------------------------------------------------------
def test_default_handle_assembles_as_before():
    ds = _ds(n_frames=90)
    a, b, c = _host(ds), _host(ds, spacing=(0.0, -1.0)), _host(ds, spacing=(10.0, 10.0))
    for h in (b, c):
        assert h.num_knots() == a.num_knots() and np.array_equal(h.imu_cells(), a.imu_cells())
        assert h.num_residuals() == a.num_residuals() and h.num_bias_prior_residuals() == 0
    assert a.num_knots()[2:] == _oracle(ds).num_knots()[2:]


@pytest.mark.parametrize("spacing", [(0.5, 0.5), (0.37, 0.23), (1.0, 0.2612)])
def test_spacing_knots_and_cells_follow_the_oracle(spacing):
    ds = _ds(n_frames=90)
    h, o = _host(ds, spacing=spacing, walk=(2e-3, 2e-4)), _oracle(ds, spacing=spacing, walk=(2e-3, 2e-4))
    assert h.num_knots() == o.num_knots()
    assert h.num_residuals() == o.num_residuals() and h.num_bias_prior_residuals() == o.num_bias_prior_residuals() > 0
    assert np.array_equal(h.imu_cells(), cells_from_segments(imu_segments(o)))
    assert h.imu_cells()[:, 2].max() > _host(ds).imu_cells()[:, 2].max()


def test_setter_arguments_and_timing():
    ds = _ds()
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    for bad in ((np.nan, 1.0), (1.0, np.inf), (1e-12, 1.0)):
        with pytest.raises(capi.IccError, match="INVALID_ARGUMENT"):
            h.set_bias_splines(*bad)
    for bad in ([1e-3, -1e-3, 1e-3], [0.0, 1e-3, 1e-3], [np.nan, 1.0, 1.0]):
        with pytest.raises(capi.IccError, match="INVALID_ARGUMENT"):
            h.set_bias_random_walk(bad, None)
        with pytest.raises(capi.IccError, match="INVALID_ARGUMENT"):
            h.set_bias_random_walk(None, bad)
    capi.load_dataset(h, ds, known_gravity=False)
    n0 = h.num_knots()
    h.set_bias_splines(0.2, 0.2); h.set_bias_random_walk(1e-3, 1e-4)
    assert h.num_knots() == n0 and h.num_bias_prior_residuals() == 0          # read by the next batch_init only
    capi.load_dataset(h, ds, known_gravity=False)
    assert h.num_knots()[2] > n0[2] and h.num_bias_prior_residuals() == 6 * (h.num_knots()[2] - 2) + 6 * (h.num_knots()[3] - 2)
    h.set_bias_random_walk(None, 1e-4); capi.load_dataset(h, ds, known_gravity=False)
    assert h.num_bias_prior_residuals() == 6 * (h.num_knots()[3] - 2)


def test_two_shards_prior_only_on_shard_zero():
    ds = _ds(n_frames=60)
    walk, sp = (2e-3, 2e-4), (0.4, 0.4)
    one = _oracle(ds, sp, walk)
    parts = [_oracle(ds, sp, walk, shard=(r, 2)) for r in range(2)]
    hosts = [_host(ds, sp, walk, shard=(r, 2)) for r in range(2)]
    assert [p.num_bias_prior_residuals() for p in parts] == [h.num_bias_prior_residuals() for h in hosts] == [one.num_bias_prior_residuals(), 0]
    rng = np.random.default_rng(9)
    so3, r3, ba, bg = one.get_knots()
    ba = ba + rng.normal(0, 0.02, ba.shape); bg = bg + rng.normal(0, 2e-3, bg.shape)
    for x in [one] + parts:
        x.set_knots(ba=ba, bg=bg)
    c1, _, g1, H1 = one.evaluate(F_BIAS, residuals=False, hessian=True)
    ev = [p.evaluate(F_BIAS, residuals=False, hessian=True) for p in parts]
    assert abs(sum(e[0] for e in ev) - c1) <= 1e-10 * c1
    np.testing.assert_allclose(sum(e[2] for e in ev), g1, rtol=1e-9, atol=1e-9 * np.abs(g1).max())
    np.testing.assert_allclose(sum(e[3] for e in ev), H1, rtol=1e-9, atol=1e-9 * np.abs(H1).max())


# ---- Allan conversion ------------------------------------------------------------------------------------------------------------------------
def _allan_doc(K):
    names = ("acc_x", "acc_y", "acc_z", "gyr_x", "gyr_y", "gyr_z")
    return {"channels": {n: {"params": {"Q": 0.0, "N": 1.0, "B": 2.0, "K": float(k), "R": 0.0}} for n, k in zip(names, K)}}


def test_allan_conversion_by_hand():
    K = [1e-3, -2e-3, 3e-3, 0.5, -0.25, 2.0]
    a, g = io_formats.bias_random_walk_from_allan(_allan_doc(K))
    np.testing.assert_array_equal(a, np.sqrt(3.0) * np.abs(K[:3]))
    np.testing.assert_array_equal(g, np.sqrt(3.0) * np.abs(K[3:]) / (57.3 * 3600))


def test_allan_conversion_recovers_the_walk():
    from allan_support import new_allan_oracle
    d = syn.make_allan_log(rate_hz=100.0, duration_s=1800.0, seed=4)
    r = new_allan_oracle().allan_variance(d["t_s"], d["accel"], d["gyro"])
    a, g = io_formats.bias_random_walk_from_allan(_allan_doc([r["params"][c][3] for c in range(6)]))
    tr = d["truth"]
    assert 1 / 3 < np.mean(a / tr["acc_walk"]) < 3 and 1 / 3 < np.mean(g / tr["gyr_walk"]) < 3, (a, g)


# ---- CLI flag rules (--parse_only) -------------------------------------------------------------------------------------------------------
def _cli_files(tmp_path):
    ds = _ds()
    return io_formats.write_dataset_files(ds, str(tmp_path))


def _run(files, *extra):
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in files.items()] + ["--parse_only"] + list(extra)
    return subprocess.run(args, capture_output=True, text=True)


def test_cli_flag_rules(tmp_path):
    files = _cli_files(tmp_path)
    plain = _run(files)
    assert plain.returncode == 0 and "bias_knot_spacing_s" not in plain.stdout
    ok = _run(files, "--reestimate_biases", "--bias_knot_spacing_s=2", "--accl_random_walk=0.002", "--gyro_random_walk=0.0002")
    assert ok.returncode == 0, ok.stderr
    s = json.loads(ok.stdout)
    assert s["bias_knot_spacing_s"] == 2.0 and s["accl_random_walk"] == [0.002] * 3 and s["gyro_random_walk"] == [0.0002] * 3
    doc = tmp_path / "noise.json"; doc.write_text(json.dumps(_allan_doc([1e-3, 2e-3, 3e-3, 0.5, 0.25, 2.0])))
    js = _run(files, "--reestimate_biases", f"--imu_noise_json={doc}")
    assert js.returncode == 0, js.stderr
    a, g = io_formats.bias_random_walk_from_allan(json.loads(doc.read_text()))
    s = json.loads(js.stdout)
    np.testing.assert_allclose(s["accl_random_walk"], a, rtol=1e-12); np.testing.assert_allclose(s["gyro_random_walk"], g, rtol=1e-12)
    for bad, msg in [(("--bias_knot_spacing_s=2",), "reestimate_biases"), (("--accl_random_walk=0.002",), "reestimate_biases"),
                     ((f"--imu_noise_json={doc}",), "reestimate_biases"),
                     (("--reestimate_biases", "--accl_random_walk=0.002", f"--imu_noise_json={doc}"), "use one"),
                     (("--reestimate_biases", "--bias_knot_spacing_s=0"), "bias_knot_spacing_s"),
                     (("--reestimate_biases", "--gyro_random_walk=-1"), "random_walk")]:
        r = _run(files, *bad)
        assert r.returncode == 1 and msg in r.stderr, (bad, r.stderr)
