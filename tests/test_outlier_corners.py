"""Outlier corners between spline solves: icc_get_corner_errors, icc_reject_outlier_corners, icc_get_corner_status and the CLI's
--outlier_sigma.  CPU: the oracle (tests/outliers/outlier_oracle.cpp) against a NumPy statement of the rule.  GPU: the product against
the oracle, and a compacted handle against a fresh handle built from the filtered inputs."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from helpers import F_STAGE1, F_STAGE2
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from openimucameracalibrator_b200 import calibrator
from outlier_support import (copy_state, filtered, inject_outliers, new_outlier_oracle, numpy_rule, outlier_sequence, reject_at, shard_worker,
                             solve_with_rejection)
from test_camera_models import CASES
from test_gpu_omni_radtan import K17, _numpy_bearings
from test_tangent_spline import set_oracle_bearings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOT_CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "continuous_time_imu_to_camera_calibration")
OMNI = (cm.OMNI_RADIAL_TANGENTIAL, np.asarray(K17, dtype=np.float64))
DP = ctypes.POINTER(ctypes.c_double)
MODELS = CASES + [OMNI]


def _ds(model=cm.DIVISION_UNDISTORTION, k=(437.1, 1.0, 489.1, 270.9, -1.44e-6), n_frames=24, **kw):
    return syn.make_dataset(syn.tiny_config(model, tuple(k), n_frames=n_frames, **kw))


def _oracle(ds, tangent=False, shard=None):
    o = new_outlier_oracle(); capi.load_dataset(o, ds, shard=shard)
    if tangent and ds["model"] == cm.OMNI_RADIAL_TANGENTIAL:   # NumPy bearings of the omni model and its pixel scale f sqrt(ar) / (1 + xi)
        k = np.asarray(ds["intrinsics"], dtype=np.float64)
        b, ok = _numpy_bearings(k, np.asarray(ds["uv"], dtype=np.float64).reshape(-1, 2))
        b = np.ascontiguousarray(b)
        o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], len(ok), b.ctypes.data_as(DP),
                ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), k[0] * np.sqrt(k[1]) / (1 + k[5]))
    elif tangent:
        set_oracle_bearings(o, ds)
    return o


def _pairs(api):
    _, r, _, _ = api.evaluate(F_STAGE1, gradient=False)
    nv, _, _ = api.num_residuals()
    return r[:nv].reshape(-1, 2)


# ---- CPU -------------------------------------------------------------------------------------------------------------------------------------
def test_oracle_errors_are_the_vision_pairs():
    ds, _ = inject_outliers(_ds())
    o = _oracle(ds)
    pairs = _pairs(o)
    e = o.corner_errors()
    assert np.array_equal(e, np.sqrt(pairs[:, 0] ** 2 + pairs[:, 1] ** 2))
    counted = (pairs[:, 0] != 0) & (pairs[:, 1] != 0)
    assert abs(e[counted].mean() - o.mean_reprojection_error()) <= 1e-12 * e[counted].mean()


@pytest.mark.parametrize("k_sigma,min_px", [(3.0, 1.0), (2.0, 0.0), (3.0, 1e3)])
def test_oracle_rejects_the_numpy_rule(k_sigma, min_px):
    """tangent mode so that a corner can fail (its bearing flipped: b.p <= 0) or give a zero pair (no bearing)"""
    ds, _ = inject_outliers(_ds())
    o = new_outlier_oracle(); capi.load_dataset(o, ds)
    b, ok = set_oracle_bearings(o, ds)
    b = b.copy(); ok = ok.copy()
    b[3] *= -1.0; ok[7] = 0                                        # one failed projection, one zero pair
    o._call("set_tangent_bearings", [ctypes.c_int, DP, ctypes.POINTER(ctypes.c_int32), ctypes.c_double], len(ok), b.ctypes.data_as(DP),
            ok.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), 437.1)
    pairs = _pairs(o)
    assert np.all(pairs[3] == 1e10) and pairs[7, 0] == 0.0
    keep, thr, rms = numpy_rule(pairs, k_sigma, min_px)
    s = o.reject_outlier_corners(k_sigma, min_px)
    assert s["threshold_px"] == pytest.approx(thr, rel=1e-12) and s["rms_px"] == pytest.approx(rms, rel=1e-12)
    assert s["n_corners"] == len(pairs) and s["n_rejected"] == int((~keep).sum()) and s["n_failed"] == 1
    st = o.corner_status()
    assert np.array_equal(st, keep.astype(np.int32))               # every frame of one shard is assembled
    assert st[3] == 0 and st[7] == 1
    assert o.num_residuals()[0] == 2 * int(keep.sum())


def test_two_shards_give_the_single_threshold_and_set():
    ds, _ = inject_outliers(_ds(n_frames=30))
    one = _oracle(ds)
    s1 = one.reject_outlier_corners(3.0, 1.0)
    shards = [_oracle(ds, shard=(r, 2)) for r in range(2)]
    pairs = [_pairs(sh) for sh in shards]
    allp = np.concatenate(pairs)
    _, thr, _ = numpy_rule(allp, 3.0, 1.0)
    assert thr == pytest.approx(s1["threshold_px"], rel=1e-12)
    for sh in shards:
        reject_at(sh, thr)
    st = [sh.corner_status() for sh in shards]
    union = np.maximum(st[0], st[1])
    assert np.array_equal(union, one.corner_status())
    assert np.all((st[0] == -1) | (st[1] == -1))


def test_oracle_after_rejection_equals_filtered_inputs():
    ds, _ = inject_outliers(_ds())
    o = _oracle(ds)
    o.lm_iterations(2, F_STAGE1)
    o.reject_outlier_corners(3.0, 1.0)
    f = _oracle(filtered(ds, o.corner_status()))
    copy_state(o, f)
    for flags in (F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_GRAVITY_DIR):
        ca, ra, ga, Ha = o.evaluate(flags, hessian=True)
        cb, rb, gb, Hb = f.evaluate(flags, hessian=True)
        assert abs(ca - cb) <= 1e-12 * abs(cb)
        assert np.array_equal(ra, rb)
        assert np.abs(ga - gb).max() <= 1e-12 * np.abs(gb).max() and np.abs(Ha - Hb).max() <= 1e-12 * np.abs(Hb).max()


def _solve(o, rounds):
    o.optimize(50, F_STAGE1)
    for _ in range(rounds):
        if o.reject_outlier_corners(3.0, 1.0)["n_rejected"] == 0:
            break
        o.optimize(50, F_STAGE1)
    o.optimize(10, F_STAGE2)
    return o.get_T_i_c(), o.get_line_delay()


def _tic_err(T, truth):
    q, qt = np.asarray(T[:4]), np.asarray(truth[:4])
    return 2 * np.arccos(min(1.0, abs(float(q @ qt)))), float(np.linalg.norm(np.asarray(T[4:]) - truth[4:]))


def test_rejection_recovers_the_clean_solve():
    clean = _ds(n_frames=40, grid=(6, 5))
    bad, idx = inject_outliers(clean, fraction=0.01)
    truth = clean["truth"]["T_i_c"]
    Tc, ldc = _solve(_oracle(clean), 0)
    Tb, _ = _solve(_oracle(bad), 0)
    o = _oracle(bad)
    Tr, ldr = _solve(o, 2)
    st = o.corner_status()
    assert np.all(st[idx] == 0)                                    # every injected outlier is gone
    db, dr = _tic_err(Tb, Tc), _tic_err(Tr, Tc)
    assert db[0] > 5e-3 and db[1] > 5e-3, db                       # without rejection T_i_c is measurably off the clean solve
    assert dr[0] < 0.1 * db[0] and dr[1] < 0.1 * db[1], (dr, db)   # after it, within a tenth of that
    assert _tic_err(Tr, truth)[1] < _tic_err(Tb, truth)[1]
    assert abs(ldr - ldc) <= 1e-3 * abs(ldc)


def test_argument_and_state_errors():
    o = new_outlier_oracle()
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        o.reject_outlier_corners(3.0, 1.0)
    ds = _ds()
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    capi.load_dataset(h, ds, known_gravity=False)
    assert np.all(h.corner_status() == 1)                          # host only: nothing rejected yet
    for k, m in ((0.0, 1.0), (-1.0, 1.0), (np.nan, 1.0), (3.0, -1.0), (3.0, np.inf), (3.0, np.nan)):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
            h.reject_outlier_corners(k, m)
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h.reject_outlier_corners(3.0, 1.0)
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h._call("get_corner_errors", [ctypes.c_int, ctypes.POINTER(ctypes.c_double)], 1, (ctypes.c_double * 1)())
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):   # no output for corners that exist
        h._call("get_corner_errors", [ctypes.c_int, ctypes.POINTER(ctypes.c_double)], 1, None)
    with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
        h._call("get_corner_status", [ctypes.c_int, ctypes.POINTER(ctypes.c_int32)], 3, (ctypes.c_int32 * 3)())


def test_cli_outlier_flags_are_parsed_and_checked(tmp_path):
    assert os.path.exists(HOT_CLI), "build the CLI first (__graft_entry__.build())"
    ds = _ds()
    paths = iof.write_dataset_files(ds, str(tmp_path))
    base = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={tmp_path}/r.json", "--parse_only"]
    plain = subprocess.run(base, capture_output=True, text=True)
    assert plain.returncode == 0 and "outlier" not in plain.stdout, plain.stderr
    on = subprocess.run(base + ["--outlier_sigma=3", "--outlier_min_px", "0.5", "--outlier_rounds=3"], capture_output=True, text=True)
    assert on.returncode == 0, on.stderr
    s = json.loads(on.stdout)
    assert s["outlier_sigma"] == 3.0 and s["outlier_min_px"] == 0.5 and s["outlier_rounds"] == 3
    for bad in ("--outlier_sigma=-1", "--outlier_min_px=-0.5", "--outlier_rounds=-1", "--outlier_sigma=nan", "--outlier_rounds=1.5"):
        r = subprocess.run(base + [bad], capture_output=True, text=True)
        assert r.returncode == 1 and "--outlier_" in r.stderr, (bad, r.stderr)


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------------
def _gpu(gpu_factory, ds, tangent=False, shard=None):
    g = gpu_factory()
    if tangent:
        g.set_reprojection_error("tangent")
    capi.load_dataset(g, ds, shard=shard)
    return g


def _pinned(ds):
    """ds with page-locked corner arrays: the product then uses them in place on the device (d_uv_all)"""
    import torch
    ds = dict(ds)
    ds["uv"] = torch.from_numpy(np.ascontiguousarray(ds["uv"], dtype=np.float64).reshape(-1, 2).copy()).pin_memory().numpy()
    ds["point_ids"] = torch.from_numpy(np.ascontiguousarray(ds["point_ids"], dtype=np.int32).copy()).pin_memory().numpy()
    return ds


def _batch_init_again(g, ds):
    """icc_batch_init_spline (and the known gravity) on the same handle, without handing it the inputs again"""
    g.batch_init_spline(ds["T_i_c_init"], ds["dt_so3_s"], ds["dt_r3_s"], ds["std_so3"], ds["std_r3"], ds["time_offset_imu_to_cam_s"],
                        ds["init_line_delay_s"], acc_bias=ds["acc_bias"], gyr_bias=ds["gyr_bias"], dispatch_fov=ds["model"] == 3)
    g.set_known_gravity_dir(ds["gravity"])


def _permute_frames(ds, perm):
    """the views of ds in the index order perm (their corners with them)"""
    off = np.asarray(ds["corner_offsets"]); uv = np.asarray(ds["uv"], dtype=np.float64).reshape(-1, 2); ids = np.asarray(ds["point_ids"])
    out = dict(ds)
    out["frame_t"] = np.asarray(ds["frame_t"])[perm]; out["q_wc"] = np.asarray(ds["q_wc"])[perm]; out["p_wc"] = np.asarray(ds["p_wc"])[perm]
    out["uv"] = np.concatenate([uv[off[i]:off[i + 1]] for i in perm]); out["point_ids"] = np.concatenate([ids[off[i]:off[i + 1]] for i in perm])
    out["corner_offsets"] = np.concatenate([[0], np.cumsum(np.diff(off)[perm])]).astype(np.int32)
    return out


def _flat(v, prefix=""):
    """numbers of a JSON tree by path"""
    if isinstance(v, dict):
        return {k2: x for k, w in v.items() for k2, x in _flat(w, f"{prefix}/{k}").items()}
    if isinstance(v, list):
        return {k2: x for i, w in enumerate(v) for k2, x in _flat(w, f"{prefix}/{i}").items()}
    return {prefix: float(v)}


def _model_ds(model, k, global_shutter=False):
    ds, _ = inject_outliers(_ds(model, k, n_frames=16))
    if global_shutter:
        ds["init_line_delay_s"] = 0.0
    return ds


@pytest.mark.gpu
@pytest.mark.parametrize("tangent", [False, True], ids=["pixel", "tangent"])
@pytest.mark.parametrize("model,k", MODELS, ids=[cm.MODEL_NAMES[m] for m, _ in MODELS])
def test_gpu_corner_errors_and_rejection_match_the_oracle(gpu_factory, model, k, tangent):
    for gs in (False, True):
        ds = _model_ds(model, k, gs)
        g, o = _gpu(gpu_factory, ds, tangent), _oracle(ds, tangent)
        if not gs:   # a moved state with the line delay and board points from the state (POINTS)
            flags = capi.FLAG_SPLINE | capi.FLAG_POINTS | capi.FLAG_CAM_LINE_DELAY
            g.lm_iterations(1, flags); o.lm_iterations(1, flags)
        eg, eo = g.corner_errors(), o.corner_errors()
        assert eg.shape == eo.shape
        assert np.all(np.abs(eg - eo) <= 1e-9 * np.maximum(np.abs(eo), 1.0)), np.abs(eg - eo).max()
        sg, so = g.reject_outlier_corners(1.0, 0.0), o.reject_outlier_corners(1.0, 0.0)   # (at the start state: a low bar, so that some go)
        assert sg["n_rejected"] == so["n_rejected"] > 0 and sg["n_failed"] == so["n_failed"] and sg["n_frames_emptied"] == so["n_frames_emptied"]
        assert sg["threshold_px"] == pytest.approx(so["threshold_px"], rel=1e-9)
        assert np.array_equal(g.corner_status(), o.corner_status())
        assert g.num_residuals() == o.num_residuals()


def _empty_one_frame(ds, frame=5):
    """every corner of one frame displaced far: the frame is emptied by the rejection"""
    ds = dict(ds); uv = np.array(ds["uv"], dtype=np.float64).reshape(-1, 2).copy()
    off = ds["corner_offsets"]; uv[off[frame]:off[frame + 1]] += 150.0
    ds["uv"] = uv
    return ds


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["host_copy", "in_place", "tangent"])
def test_gpu_compacted_handle_equals_fresh_filtered_handle(gpu_factory, path, eval_path):
    """host_copy: pageable inputs, the used corners copied up from the host; in_place: page-locked inputs used where set_frames put them"""
    ds, _ = inject_outliers(_ds(n_frames=24))
    ds = _empty_one_frame(ds)
    if path == "in_place":
        ds = _pinned(ds)
    given = {k: np.array(ds[k], copy=True) for k in ("uv", "point_ids")}
    tangent = path == "tangent"
    g = _gpu(gpu_factory, ds, tangent)
    g.lm_iterations(2, F_STAGE1)
    s = g.reject_outlier_corners(3.0, 1.0)
    assert s["n_frames_emptied"] == 1 and s["n_rejected"] > 0
    st = g.corner_status()
    f = _gpu(gpu_factory, filtered(ds, st), tangent)
    copy_state(g, f)
    a, b = g.eval_schedule(), f.eval_schedule()
    assert a["n_vchunks"] == b["n_vchunks"] and a["n_ichunks"] == b["n_ichunks"]
    assert np.array_equal(a["vitems"], b["vitems"]) and np.array_equal(a["iitems"], b["iitems"])
    assert g.num_residuals() == f.num_residuals()
    for flags in (F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_GRAVITY_DIR):
        ca, ra, ga, Ha = g.evaluate(flags, hessian=True)
        cb, rb, gb, Hb = f.evaluate(flags, hessian=True)
        assert np.array_equal(ra, rb)
        assert abs(ca - cb) <= 1e-12 * abs(cb)
        assert np.abs(ga - gb).max() <= 1e-12 * np.abs(gb).max() and np.abs(Ha - Hb).max() <= 1e-12 * np.abs(Hb).max()
    # the inputs stay as given: batch_init alone (no set_frames) assembles every corner again, equal to a fresh handle of the same inputs
    assert all(np.array_equal(np.asarray(ds[k]), given[k]) for k in given)
    _batch_init_again(g, ds)
    assert np.all(g.corner_status() == 1)
    fresh = _gpu(gpu_factory, ds, tangent)
    assert g.num_residuals() == fresh.num_residuals()
    assert np.array_equal(g.evaluate(F_STAGE1, gradient=False)[1], fresh.evaluate(F_STAGE1, gradient=False)[1])


@pytest.mark.gpu
def test_gpu_gathered_corners_match_the_oracle(gpu_factory):
    """views out of time order in shard 0 of 2: the shard's views are not one index run, so its corners are gathered on the host (used_uv)"""
    ds, _ = inject_outliers(_ds(n_frames=30))
    perm = np.random.default_rng(3).permutation(len(ds["frame_t"]))
    ds = _empty_one_frame(_permute_frames(ds, perm), frame=5)
    g, o = _gpu(gpu_factory, ds, shard=(0, 2)), _oracle(ds, shard=(0, 2))
    here = np.flatnonzero([(g.corner_status()[ds["corner_offsets"][i]:ds["corner_offsets"][i + 1]] != -1).any() for i in range(len(perm))])
    assert 5 in here and np.any(np.diff(here) > 1)                  # view 5 is in the shard, whose views are not one contiguous run
    g.lm_iterations(2, F_STAGE1); o.lm_iterations(2, F_STAGE1)
    sg, so = g.reject_outlier_corners(1.0, 0.0), o.reject_outlier_corners(1.0, 0.0)   # (an early state: a low bar, so that some go)
    assert sg["n_rejected"] == so["n_rejected"] > 0 and sg["n_frames_emptied"] == so["n_frames_emptied"] >= 1
    assert np.array_equal(g.corner_status(), o.corner_status())
    assert g.num_residuals() == o.num_residuals()
    for flags in (F_STAGE1, F_STAGE1 | capi.FLAG_CAM_LINE_DELAY | capi.FLAG_GRAVITY_DIR):
        cg, rg, gg, Hg = g.evaluate(flags, hessian=True)
        co, ro, go, Ho = o.evaluate(flags, hessian=True)
        assert abs(cg - co) <= 1e-9 * abs(co) and np.abs(rg - ro).max() <= 1e-9 * np.abs(ro).max()
        assert np.abs(gg - go).max() <= 1e-9 * np.abs(go).max() and np.abs(Hg - Ho).max() <= 1e-9 * np.abs(Ho).max()


def _run_shards(tmp_path, mode):
    import torch.multiprocessing as mp
    port = 31000 + (os.getpid() % 2000) + 7 * ["gloo", "nccl_hook", "native"].index(mode)
    mp.spawn(shard_worker, args=(2, port, str(tmp_path), mode), nprocs=2, join=True)
    return [np.load(tmp_path / f"status{r}.npy") for r in range(2)], [np.load(tmp_path / f"summary{r}.npy") for r in range(2)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["gloo", "nccl_hook", "native"])
def test_gpu_sharded_rejection_equals_single_gpu(tmp_path, gpu_factory, mode):
    """Two ranks: "gloo" shares device 0 (the cross-rank sums through the caller hook, on the host), "nccl_hook" / "native" need 2 GPUs.
    Both ranks report the same summary, with the single-GPU threshold and counts; their status arrays are disjoint and their union is the
    single-GPU status; the re-solve follows the single-GPU LM path."""
    import torch
    if mode != "gloo" and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    st, sm = _run_shards(tmp_path, mode)
    pairs = np.concatenate([np.load(tmp_path / f"pairs{r}.npy") for r in range(2)])
    g = gpu_factory(); capi.load_dataset(g, outlier_sequence())
    s, iters, _ = solve_with_rejection(g)
    # every rank reports the summed counts and the one threshold; each rank keeps its own copy of the state, which the ranks' solves
    # (atomic sums inside) may leave a few ulps apart
    assert np.array_equal(sm[0][[0, 1, 2, 3, 6]], sm[1][[0, 1, 2, 3, 6]])
    assert np.abs(sm[0][4:6] - sm[1][4:6]).max() <= 1e-12 * sm[0][5] and np.abs(sm[0][7:] - sm[1][7:]).max() <= 1e-12
    # the threshold is the rule over both shards' pairs together
    keep, thr, rms = numpy_rule(pairs, 3.0, 1.0)
    assert sm[0][5] == pytest.approx(thr, rel=1e-12) and sm[0][4] == pytest.approx(rms, rel=1e-12) and sm[0][1] == int((~keep).sum())
    assert sm[0][0] == len(pairs) == s["n_corners"] and sm[0][1] == s["n_rejected"] > 0 and sm[0][2] == s["n_failed"] and sm[0][3] == s["n_frames_emptied"]
    # the single-GPU run reaches the rejection at a state within the sharded LM's ~1e-8 of it
    assert sm[0][5] == pytest.approx(s["threshold_px"], rel=1e-6)
    assert np.all((st[0] == -1) | (st[1] == -1)) and (st[0] == -1).any() and (st[1] == -1).any()
    assert np.array_equal(np.maximum(st[0], st[1]), g.corner_status())
    # the same LM iterations on the reduced set.  On 40 views T_i_c is weakly determined: sharded and single solves that agree in cost and
    # threshold to ~1e-8 sit ~1e-5 apart in T_i_c, so this only shows both land on the same solution
    dT = np.abs(sm[0][7:] - g.get_T_i_c()).max()
    assert sm[0][6] == iters == 10 and dT <= 1e-4, dT


@pytest.mark.gpu
def test_gpu_cli_outlier_sigma_on_two_gpus(tmp_path):
    """--gpus 2 --outlier_sigma 3 (one rank process per device, every round's sums over NCCL) writes what --gpus 1 writes"""
    import signal
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ds = outlier_sequence()
    res = []
    for gpus in (1, 2):
        d = tmp_path / f"g{gpus}"; d.mkdir()
        paths = iof.write_dataset_files(ds, str(d))
        args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + [f"--result_output_json={d}/result.json", "--known_grav_dir_axis", "Z",
                                                                          "--outlier_sigma", "3", f"--gpus={gpus}"]
        proc = subprocess.Popen(args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
        try:
            so, se = proc.communicate(timeout=120)
        except subprocess.TimeoutExpired:
            os.killpg(proc.pid, signal.SIGKILL)
            so, se = proc.communicate()
            pytest.fail(f"--gpus={gpus} did not finish in 120 s\n{so[-2000:]}\n{se[-2000:]}")
        assert proc.returncode == 0, se + so
        res.append(json.loads(open(d / "result.json").read()))
    a, b = res
    assert a["outlier_corners_rejected"] == b["outlier_corners_rejected"] > 0
    assert a["outlier_threshold_px"] == pytest.approx(b["outlier_threshold_px"], rel=1e-9)
    for k in "xyz":
        assert abs(a["t_i_c"][k] - b["t_i_c"][k]) < 1e-8


@pytest.mark.gpu
def test_gpu_lm_after_rejection_matches_the_oracle(gpu_factory):
    ds, _ = inject_outliers(_ds(n_frames=24))
    g, o = _gpu(gpu_factory, ds), _oracle(ds)
    g.optimize(50, F_STAGE1); o.optimize(50, F_STAGE1)
    assert g.reject_outlier_corners(3.0, 1.0)["n_rejected"] == o.reject_outlier_corners(3.0, 1.0)["n_rejected"]
    sg, so = g.optimize(50, F_STAGE1), o.optimize(50, F_STAGE1)
    assert sg.iterations == so.iterations
    assert np.abs(g.get_T_i_c() - o.get_T_i_c()).max() <= 1e-8


@pytest.mark.gpu
def test_gpu_full_size_config4_rejection_round():
    from openimucameracalibrator_b200 import calibrator
    ds, idx = inject_outliers(syn.make_dataset(syn.CONFIGS[4]))
    g = capi.CApi(calibrator.load_library(), "icc_", 0); capi.load_dataset(g, ds)
    g.optimize(5, F_STAGE1)
    s = g.reject_outlier_corners(3.0, 1.0)
    assert s["n_corners"] == len(ds["point_ids"]) and s["n_rejected"] >= len(idx)
    assert np.all(g.corner_status()[idx] == 0)
    g.optimize(3, F_STAGE1)


@pytest.mark.gpu
def test_gpu_cli_outlier_sigma(tmp_path):
    clean = _ds(n_frames=40, grid=(6, 5))
    ds, _ = inject_outliers(clean)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    base = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items()] + ["--known_grav_dir_axis", "Z"]
    out = {}
    for name, extra in (("off", []), ("off2", []), ("zero", ["--outlier_sigma=0"]), ("on", ["--outlier_sigma", "3"])):
        r = subprocess.run(base + [f"--result_output_json={tmp_path}/{name}.json"] + extra, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out[name] = r
    raw = {n: open(f"{tmp_path}/{n}.json", "rb").read() for n in out}
    # without the flag nothing of the rejection runs: the file equals the one written with --outlier_sigma 0 -- byte for byte when two
    # runs of the same command agree byte for byte; the device's atomic sums may reorder from run to run, and 50 LM iterations carry that
    # into the last digits, so otherwise every key is the same and every value agrees as closely as the two plain runs agree
    if raw["off"] == raw["off2"]:
        assert raw["off"] == raw["zero"]
    else:
        fa, f2, fz = (_flat(json.loads(raw[n])) for n in ("off", "off2", "zero"))
        assert fa.keys() == fz.keys() == f2.keys()
        spread = max(abs(fa[k] - f2[k]) / max(1.0, abs(fa[k])) for k in fa)
        worst = max(abs(fa[k] - fz[k]) / max(1.0, abs(fa[k])) for k in fa)
        assert worst <= max(1e-9, 10 * spread), (worst, spread)
    assert "Outlier round 1" in out["on"].stdout
    res = {n: json.loads(raw[n]) for n in ("off", "on")}
    assert "outlier_corners_rejected" not in res["off"] and res["on"]["outlier_corners_rejected"] > 0 and res["on"]["outlier_threshold_px"] > 0
    truth = clean["truth"]["T_i_c"]
    t = {n: np.array([res[n]["t_i_c"][a] for a in "xyz"]) for n in res}
    assert np.linalg.norm(t["on"] - truth[4:]) < np.linalg.norm(t["off"] - truth[4:])
