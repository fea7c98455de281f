"""Bias-spline spacing and the random-walk prior on the GPU against the oracle (tests/bias_walk/bias_walk_oracle.cpp): cost, residuals, J^T r
and J^T J of the prior kernel (icc_bias_prior.cu), the unchanged default path, the LM, the border limit at BASELINE config 4, sharding,
recovery of drifting biases and the hot CLI chain from an Allan fit."""
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

from bias_walk_support import DRIFT, drifting_dataset, new_bias_walk_oracle, prior_rows_of
from openimucameracalibrator_b200 import _capi as capi, calibrator, io_formats, synthetic as syn
from scaled_parity import assert_block_probes, assert_scaled_parity, probe_reference
from test_tangent_spline import set_oracle_bearings

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")
F1 = capi.FLAG_SPLINE | capi.FLAG_T_I_C
F_BIAS = F1 | capi.FLAG_IMU_BIASES
WALK = {"acc": ((2e-3, 3e-3, 1e-3), None), "gyr": (None, (1e-4, 2e-4, 3e-4)), "both": ((2e-3, 3e-3, 1e-3), (1e-4, 2e-4, 3e-4))}
FLAGS = {"free": F_BIAS, "fixed": F1}


def _seq(spacing):
    if spacing < 1.0:   # short sequence (0.8 s): several knots at 0.5 s
        return syn.make_dataset(syn.tiny_config(n_frames=24))
    return syn.make_dataset(syn.tiny_config(n_frames=600, grid=(4, 3), dt_so3_s=0.2, dt_r3_s=0.2))   # 20 s


def _pair(ds, spacing, walk, tangent=False, shard=None):
    g = capi.CApi(calibrator.load_library(), "icc_", 0)
    o = new_bias_walk_oracle()
    for x in (g, o):
        x.set_bias_splines(spacing, spacing)
        x.set_bias_random_walk(*walk)
    if tangent:
        g.set_reprojection_error(capi.REPROJ_ERROR_TANGENT)
    capi.load_dataset(g, ds, shard=shard); capi.load_dataset(o, ds, shard=shard)
    if tangent:
        set_oracle_bearings(o, ds)
    return g, o


def _perturb(g, o, seed=1):
    """biases away from the start value, so that every prior row is non-zero"""
    rng = np.random.default_rng(seed)
    _, _, ba, bg = o.get_knots()
    ba = ba + rng.normal(0, 0.02, ba.shape); bg = bg + rng.normal(0, 2e-3, bg.shape)
    for x in (g, o):
        x.set_knots(ba=ba, bg=bg)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("tangent", [False, True], ids=["pixel", "tangent"])
@pytest.mark.parametrize("free", list(FLAGS))
@pytest.mark.parametrize("sensors", list(WALK))
@pytest.mark.parametrize("spacing", [10.0, 2.0, 0.5])
def test_prior_parity_dense(spacing, sensors, free, tangent):
    ds = _seq(spacing)
    g, o = _pair(ds, spacing, WALK[sensors], tangent)
    _perturb(g, o)
    assert g.num_bias_prior_residuals() == o.num_bias_prior_residuals() > 0
    cg, rg, gg, Hg = g.evaluate(FLAGS[free], hessian=True)
    co, ro, go, Ho = o.evaluate(FLAGS[free], hessian=True)
    assert abs(cg - co) <= 1e-9 * abs(co)
    assert _rel(rg, ro) < 1e-9 and _rel(gg, go) < 1e-9 and _rel(Hg, Ho) < 1e-9
    assert_scaled_parity(g, FLAGS[free], (co, ro, go, Ho), (cg, rg, gg, Hg))      # the prior rows and bias columns at their own scale
    nres = sum(g.num_residuals())
    assert np.abs(rg[nres:]).min() > 0.0
    cc, rc, _, _ = g.evaluate(FLAGS[free], gradient=False)                  # the cost-only kernel path
    assert abs(cc - co) <= 1e-9 * abs(co) and _rel(rc, ro) < 1e-9


def test_default_path_is_bit_identical():
    ds = _seq(10.0)
    a = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(a, ds)
    b = capi.CApi(calibrator.load_library(), "icc_", 0); b.set_bias_splines(10.0, 10.0); b.set_bias_random_walk(None, None); capi.load_dataset(b, ds)
    for flags in (F1, F_BIAS):
        ra, rb = a.evaluate(flags, gradient=False)[1], b.evaluate(flags, gradient=False)[1]
        assert np.array_equal(ra, rb) and b.num_bias_prior_residuals() == 0
        ja, jb = a.evaluate(flags, hessian=True), b.evaluate(flags, hessian=True)
        assert np.array_equal(ja[1], jb[1])


def test_two_stage_lm_against_the_oracle():
    ds = _seq(2.0)
    g, o = _pair(ds, 2.0, WALK["both"])
    for flags in (F1, F_BIAS):
        sg, so = g.optimize(50, flags), o.optimize(50, flags)
        assert sg.iterations == so.iterations and sg.successful_steps == so.successful_steps
        assert sg.num_residuals == so.num_residuals == sum(g.num_residuals()) + g.num_bias_prior_residuals()
        assert abs(sg.final_cost - so.final_cost) <= 1e-8 * so.final_cost
        assert np.abs(g.get_T_i_c() - o.get_T_i_c()).max() < 1e-8


def test_config4_normal_equations_and_border_limit():
    ds = syn.make_dataset(syn.CONFIGS[4])
    g, o = _pair(ds, 2.0, WALK["both"])
    _perturb(g, o)
    n = g.num_tangent(F_BIAS)
    rng = np.random.default_rng(5)
    V = rng.standard_normal((3, n))
    Vb = np.zeros((1, n)); Vb[0, n - 6 * g.num_knots()[2]:] = 1.0              # the bias columns (last in the canonical order here)
    V = np.concatenate([V, Vb])
    assert _rel(g.normal_matvec(F_BIAS, V), o.normal_matvec(F_BIAS, V)) < 1e-9
    assert_block_probes(g, probe_reference(o, F_BIAS, rng))
    assert abs(g.evaluate(F_BIAS, residuals=False, gradient=False)[0] - o.evaluate(F_BIAS, residuals=False, gradient=False)[0]) <= 1e-9 * o.evaluate(F_BIAS, residuals=False, gradient=False)[0]
    s = g.lm_iterations(2, F_BIAS)                                              # 2 s: 2 * 3 * 52 + 6 = 318 border columns, solved
    assert s.iterations == 2 and np.isfinite(s.final_cost)
    # 1 s: 618 border columns, refused, the state untouched
    h = capi.CApi(calibrator.load_library(), "icc_", 0); h.set_bias_splines(1.0, 1.0); capi.load_dataset(h, ds)
    before = h.get_knots(), h.get_T_i_c()
    with pytest.raises(capi.IccError, match=r"UNSUPPORTED.*bias knots: 102 accelerometer knots at 1 s spacing, 102 gyroscope knots"):
        h.lm_iterations(1, F_BIAS)
    after = h.get_knots(), h.get_T_i_c()
    assert all(np.array_equal(x, y) for x, y in zip(before[0], after[0])) and np.array_equal(before[1], after[1])


def _shard_worker(rank, world, port, out_dir):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from openimucameracalibrator_b200.distributed import DevicePointer
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ds = _seq(2.0)
    g = capi.CApi(calibrator.load_library(), "icc_", 0)
    g.set_bias_splines(2.0, 2.0); g.set_bias_random_walk(*WALK["both"])
    capi.load_dataset(g, ds, shard=(rank, world))
    ext = torch.cuda.ExternalStream(g.get_stream(), device="cuda:0")

    def hook(ptr, n, stream, user):
        t = torch.as_tensor(DevicePointer(ptr, n), device="cuda:0")
        ext.synchronize(); h = t.cpu(); dist.all_reduce(h); t.copy_(h); torch.cuda.synchronize(0)
    g.set_allreduce(hook)
    c, _, gr, H = g.evaluate(F_BIAS, residuals=False, hessian=True)
    s = g.lm_iterations(5, F_BIAS)
    np.save(os.path.join(out_dir, f"r{rank}.npy"), np.concatenate([[c, s.final_cost, g.num_bias_prior_residuals()], gr, H.ravel(), g.get_T_i_c()]))
    g.close(); dist.destroy_process_group()


def test_two_gloo_shards_equal_one_gpu():
    import torch.multiprocessing as mp
    d = tempfile.mkdtemp(prefix="icc_bw_shards_")
    mp.spawn(_shard_worker, args=(2, 29671, d), nprocs=2, join=True)
    r0, r1 = np.load(os.path.join(d, "r0.npy")), np.load(os.path.join(d, "r1.npy"))
    g = capi.CApi(calibrator.load_library(), "icc_", 0); g.set_bias_splines(2.0, 2.0); g.set_bias_random_walk(*WALK["both"]); capi.load_dataset(g, _seq(2.0))
    c, _, gr, H = g.evaluate(F_BIAS, residuals=False, hessian=True)
    s = g.lm_iterations(5, F_BIAS)
    one = np.concatenate([[c, s.final_cost, g.num_bias_prior_residuals()], gr, H.ravel(), g.get_T_i_c()])
    assert r0[2] == one[2] and r1[2] == 0
    for r in (r0, r1):
        assert _rel(r[3:], one[3:]) < 1e-9 and abs(r[0] - one[0]) <= 1e-10 * one[0] and abs(r[1] - one[1]) <= 1e-9 * one[1]


def _bias_rms(g, ds):
    tr = ds["bias_truth"]
    t_ns = (tr["t_cam"] * 1e9).astype(np.int64)
    out = g.eval_trajectory(t_ns)
    keep = (tr["t_cam"] >= ds["frame_t"][0]) & (tr["t_cam"] < ds["frame_t"][-1])
    return (float(np.sqrt(np.mean((out["accel_bias"][keep] - tr["acc"][keep]) ** 2))), float(np.sqrt(np.mean((out["gyro_bias"][keep] - tr["gyr"][keep]) ** 2))))


def _tic_error(g, ds):
    T, T0 = g.get_T_i_c(), ds["truth"]["T_i_c"]
    q, q0 = T[:4] / np.linalg.norm(T[:4]), T0[:4]
    ang = 2 * np.arccos(min(1.0, abs(float(np.dot(q, q0)))))
    return ang, float(np.linalg.norm(T[4:] - T0[4:]))


def test_drifting_biases_are_recovered():
    ds = drifting_dataset()
    res = {}
    for name, spacing, walk in (("reference", 10.0, (None, None)), ("prior", 2.0, (DRIFT["acc_q"], DRIFT["gyr_q"]))):
        g = capi.CApi(calibrator.load_library(), "icc_", 0)
        g.set_bias_splines(spacing, spacing); g.set_bias_random_walk(*walk)
        capi.load_dataset(g, ds)
        g.optimize(50, F1); g.optimize(50, F_BIAS)
        res[name] = _bias_rms(g, ds) + _tic_error(g, ds)
    print("bias-recovery (acc rms, gyr rms, T_i_c angle rad, T_i_c translation m):", res)
    ref, pri = res["reference"], res["prior"]
    # measured on an H100: accelerometer 0.0352 vs 0.0365 m/s^2, gyroscope 1.48e-3 vs 1.78e-3 rad/s, T_i_c 4.0e-3 vs 4.1e-3 rad and
    # 3.87 vs 3.88 mm (prior vs reference)
    assert pri[0] < 0.99 * ref[0] and pri[1] < 0.9 * ref[1], res
    assert pri[2] <= 1.05 * ref[2] and pri[3] <= 1.05 * ref[3], res


def test_cli_chain_from_an_allan_fit(tmp_path):
    d = syn.make_allan_log(rate_hz=200.0, duration_s=600.0, seed=6)
    tel = tmp_path / "static.json"
    tel.write_text(json.dumps({"timestamps_ns": np.round(d["t_s"] * 1e9).tolist(), "accelerometer": d["accel"].tolist(), "gyroscope": d["gyro"].tolist()}))
    noise = tmp_path / "noise.json"
    subprocess.run([os.path.join(BIN, "fit_allan_variance"), f"--telemetry_json={tel}", f"--output_json={noise}"], check=True, capture_output=True)
    acc_q, gyr_q = io_formats.bias_random_walk_from_allan(json.loads(noise.read_text()))
    ds = syn.make_dataset(syn.tiny_config(n_frames=300))
    paths = io_formats.write_dataset_files(ds, str(tmp_path))
    base = [os.path.join(BIN, "continuous_time_imu_to_camera_calibration")] + [f"--{a}={b}" for a, b in paths.items()] + ["--reestimate_biases"]

    def run(out, *extra):
        r = subprocess.run(base + [f"--result_output_json={tmp_path / out}"] + list(extra), capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        return r.stdout, json.loads((tmp_path / out).read_text()), (tmp_path / out).read_bytes()
    out1, res1, _ = run("r1.json", f"--imu_noise_json={noise}", "--bias_knot_spacing_s=2")
    assert "Bias splines:" in out1 and "at 2 s spacing" in out1
    assert res1["bias_knot_spacing_s"] == 2.0
    np.testing.assert_allclose(res1["accl_random_walk"], acc_q, rtol=1e-12); np.testing.assert_allclose(res1["gyro_random_walk"], gyr_q, rtol=1e-12)
    # without the flags: the keys of a default run, and its values (two runs of the solve agree to rounding, not bit for bit: the
    # evaluation kernels sum with atomics)
    _, res0, _ = run("p1.json")
    _, res0b, _ = run("p2.json")
    assert set(res0) == set(res0b) and not {"bias_knot_spacing_s", "accl_random_walk", "gyro_random_walk"} & set(res0)
    for k in ("q_i_c", "t_i_c"):
        for a in res0[k]:
            assert abs(res0[k][a] - res0b[k][a]) < 1e-9
    import torch
    if torch.cuda.device_count() >= 2:
        _, res2, _ = run("r2.json", f"--imu_noise_json={noise}", "--bias_knot_spacing_s=2", "--gpus=2")
        for k in ("q_i_c", "t_i_c"):
            for a in res1[k]:
                assert abs(res2[k][a] - res1[k][a]) < 1e-7
        assert res2["accl_random_walk"] == res1["accl_random_walk"]
