"""The C-ABI library loads, exports every symbol include/icc_b200.h declares, refuses to compute without a GPU, and its
host-side problem assembly (BatchInitSpline) agrees with the oracle's restatement of the reference."""
import ctypes
import os
import re

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import calibrator
from openimucameracalibrator_b200 import synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "icc_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(icc_[a-z0-9_]+)\s*\(", text)) - {"icc_allreduce_fn"})


def test_library_exports_every_declared_symbol():
    lib = calibrator.load_library()
    syms = _declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/icc_b200.h but not exported"


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the no-device path is exercised on the CPU box")
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        capi.CApi(calibrator.load_library(), "icc_", 0)
    # a host-only handle can assemble but must refuse every compute entry point
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    capi.load_dataset(h, syn.make_dataset(syn.tiny_config()))
    for call in (lambda: h.optimize(1, 66), lambda: h.evaluate(66), lambda: h.lm_iterations(1, 66), lambda: h.mean_reprojection_error(),
                 lambda: h.eval_trajectory([0]), lambda: h.time_evaluations(1, 66),
                 lambda: h.calibrate_camera(0, 960, 540, [0, 1], [0], [[1.0, 2.0]]), lambda: h.estimate_imu_biases(np.ones((4, 3)), np.ones((4, 3))),
                 lambda: h.optimize_board_points([0, 1], [0], [[1.0, 2.0]], [[0, 0, 0, 1.0]], [[0, 0, 1.0]], [1])):
        with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
            call()


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(calibrator, "_LIB", None)
    monkeypatch.setattr(calibrator, "library_path", lambda: str(tmp_path / "libicc_b200.so"))
    with pytest.raises(capi.IccError, match="no CPU fallback"):
        calibrator.load_library()


def test_product_package_never_references_the_oracle():
    pkg = os.path.join(ROOT, "openimucameracalibrator_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                assert "libicc_oracle" not in text and "icc_oracle" not in text and "oracle_api" not in text and "icco_" not in text.replace("`icco_`", ""), f


@pytest.mark.parametrize("cfg", [syn.tiny_config(), syn.tiny_config(dt_so3_s=0.04, dt_r3_s=0.07), syn.CONFIGS[1]], ids=["tiny", "tiny_uneven_dt", "cfg1"])
def test_host_assembly_matches_oracle(oracle_factory, cfg):
    """Knot counts, knot initialisation (slerp/lerp quirks), kept IMU samples, residual counts, gravity init."""
    ds = syn.make_dataset(cfg)
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    h = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(h, ds, known_gravity=False)
    assert o.num_knots() == h.num_knots()
    assert o.num_residuals() == h.num_residuals()
    for a, b in zip(o.get_knots(), h.get_knots()):
        assert np.array_equal(a, b) or np.allclose(a, b, rtol=0, atol=1e-15)
    for a, b in zip(o.imu_used(), h.imu_used()):
        assert np.array_equal(a, b)
    assert np.allclose(o.get_gravity(), h.get_gravity(), rtol=0, atol=1e-14)
    assert np.allclose(o.get_T_i_c(), h.get_T_i_c(), rtol=0, atol=1e-15)
    for flags in (66, 66 | 16 | 32 | 4, 32, 66 | 8, 8, 66 | 1, 1):      # | 1 = POINTS: three tangent columns per board point
        assert o.num_tangent(flags) == h.num_tangent(flags)
    assert h.num_tangent(66 | 1) == h.num_tangent(66) + 3 * len(ds["board_xyzw"])
    with pytest.raises(capi.IccError, match="UNSUPPORTED"):
        h.num_tangent(66 | 1 | capi.FLAG_CAM_INTRINSICS)   # POINTS with this library's camera-intrinsics extension


def test_shards_partition_the_residuals(oracle_factory):
    ds = syn.make_dataset(syn.tiny_config())
    full = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(full, ds)
    tot = np.zeros(3, dtype=int)
    for r in range(3):
        h = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(h, ds, shard=(r, 3))
        o = oracle_factory(); capi.load_dataset(o, ds, shard=(r, 3))
        assert h.num_residuals() == o.num_residuals()
        tot += np.array(h.num_residuals())
    assert tuple(tot) == full.num_residuals()


def test_invalid_arguments_are_reported():
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    with pytest.raises(capi.IccError, match="INVALID_ARGUMENT"):
        h.set_camera(4, [1.0, 2.0], 10, 10)           # wrong intrinsic count
    with pytest.raises(capi.IccError, match="STATE"):
        h.batch_init_spline(np.array([0, 0, 0, 1, 0, 0, 0.0]), 0.05, 0.05, 1, 1, 0, 1e-5)
    with pytest.raises(capi.IccError, match="INVALID_ARGUMENT"):
        h.set_shard(3, 2)


@pytest.mark.parametrize("case", ["shuffled_imu", "imu_hole", "duplicate_view_time"])
def test_host_assembly_general_paths_match_oracle(oracle_factory, case):
    """The one-shard fast path of BatchInitSpline assumes a time-sorted, gap-free IMU stream and increasing view timestamps; anything
    else must fall back to the general path and still agree with the oracle."""
    ds = dict(syn.make_dataset(syn.tiny_config()))
    if case == "shuffled_imu":
        perm = np.random.default_rng(0).permutation(len(ds["imu_t"]))
        ds["imu_t"], ds["accel"], ds["gyro"] = ds["imu_t"][perm], ds["accel"][perm], ds["gyro"][perm]
    elif case == "imu_hole":
        t = ds["imu_t"].copy(); t[50] = 1e6; ds["imu_t"] = t            # one sample far outside the window, mid-stream
    else:
        t = ds["frame_t"].copy(); t[5] = t[4]; ds["frame_t"] = t
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    h = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(h, ds, known_gravity=False)
    assert o.num_residuals() == h.num_residuals() and o.num_knots() == h.num_knots()
    for a, b in zip(o.imu_used(), h.imu_used()):
        assert np.array_equal(a, b)
    for a, b in zip(o.get_knots(), h.get_knots()):
        assert np.allclose(a, b, rtol=0, atol=1e-15)
    assert np.allclose(o.get_gravity(), h.get_gravity(), rtol=0, atol=1e-14)


def calc_times_cells(ds, t_used):
    """NumPy statement of CalcTimes' knot-interval cells (impl.h:763-788) of the kept samples t_used (offset-corrected, as imu_used()
    returns them): st = int64((t + offset) 1e9) - int64(min(frame_t) 1e9), the segment indices st // dt of the SO(3), R^3 and both bias
    splines (bias knots every 10 s), and cells = maximal runs of equal index tuples -> rows (s_so3, s_r3, s_acc_bias, s_gyr_bias, i_begin, i_end)."""
    st = (np.asarray(t_used) * 1e9).astype(np.int64) - np.int64(np.min(ds["frame_t"]) * 1e9)
    dts = (np.int64(ds["dt_so3_s"] * 1e9), np.int64(ds["dt_r3_s"] * 1e9), np.int64(10 * 10**9), np.int64(10 * 10**9))
    seg = np.stack([st // dt for dt in dts], axis=1).reshape(-1, 4)
    if len(seg) == 0:
        return np.zeros((0, 6), dtype=np.int32)
    bounds = np.concatenate([[0], np.flatnonzero(np.any(seg[1:] != seg[:-1], axis=1)) + 1, [len(seg)]])
    return np.column_stack([seg[bounds[:-1]], bounds[:-1], bounds[1:]]).astype(np.int32)


def _irregular_sorted_stream(dts):
    """A time-sorted IMU stream at four times the rate with irregular stamps, stamps exactly on knot boundaries of either spline and
    repeated stamps, reaching 0.2 s past the frames on both sides."""
    ds = dict(syn.make_dataset(syn.tiny_config(n_frames=40, dt_so3_s=dts[0], dt_r3_s=dts[1])))
    rng = np.random.default_rng(int(1000 * dts[0]))
    t0 = float(ds["frame_t"][0]) - ds["time_offset_imu_to_cam_s"]
    n = 4 * len(ds["imu_t"])
    t = np.sort(rng.uniform(ds["imu_t"][0] - 0.2, ds["imu_t"][-1] + 0.2, size=n))
    k = np.arange(0, n, 7); t[k] = t0 + dts[0] * np.round((t[k] - t0) / dts[0])
    k = np.arange(3, n, 11); t[k] = t0 + dts[1] * np.round((t[k] - t0) / dts[1])
    t = np.sort(t); t[5::13] = t[4::13][: len(t[5::13])]; t = np.sort(t)
    ds["imu_t"] = t; ds["accel"] = rng.normal(size=(n, 3)); ds["gyro"] = rng.normal(size=(n, 3))
    return ds


def _unsorted_copy(ds):
    """The same stream with one more sample, far before the window, appended at its end: no longer sorted (the general selection),
    same kept samples, still one contiguous run of the input."""
    ds = dict(ds)
    ds["imu_t"] = np.append(ds["imu_t"], ds["imu_t"][0] - 100.0)
    ds["accel"] = np.vstack([ds["accel"], ds["accel"][:1]]); ds["gyro"] = np.vstack([ds["gyro"], ds["gyro"][:1]])
    return ds


def _host_assembly(ds, shard=None):
    h = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(h, ds, known_gravity=False, shard=shard)
    s = h.eval_schedule()
    out = dict(used=h.imu_used(), cells=h.imu_cells(), res=h.num_residuals(),
               schedule=(s["n_vchunks"], s["n_ichunks"], s["vitems"].tolist(), s["iitems"].tolist()))
    h.close()
    return out


def _assert_same_assembly(a, b):
    assert a["res"] == b["res"] and a["schedule"] == b["schedule"]
    assert np.array_equal(a["cells"], b["cells"])
    for x, y in zip(a["used"], b["used"]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dts", [(0.05, 0.05), (0.04, 0.07), (0.09, 0.05)])
def test_imu_cells_by_bisection_equal_calc_times_cells(dts):
    """BatchInitSpline finds the knot-interval cells of a time-sorted IMU stream by galloping + bisection for the next interval boundary:
    they are CalcTimes' cells of the kept samples, and the sample-by-sample selection of an unsorted copy keeps the same samples in the same
    cells -- for irregular stamps, stamps exactly on knot boundaries of either spline and repeated stamps."""
    ds = _irregular_sorted_stream(dts)
    a, b = _host_assembly(ds), _host_assembly(_unsorted_copy(ds))
    _assert_same_assembly(a, b)
    cells, t_used = a["cells"], a["used"][0]
    assert len(cells) > 10
    assert np.array_equal(cells, calc_times_cells(ds, t_used))
    assert cells[0, 4] == 0 and cells[-1, 5] == len(t_used) and np.array_equal(cells[1:, 4], cells[:-1, 5])     # the cells tile the kept samples


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_sorted_and_general_selection_agree_on_every_shard(world):
    """Every shard of a time-sorted stream (selected on counts) equals the same shard of the unsorted copy (time merge + shard rule):
    kept samples, cells, residual counts and the persistent kernel's schedule; its cells are CalcTimes', and the shards tile the
    one-shard selection."""
    ds = _irregular_sorted_stream((0.04, 0.07))
    full = _host_assembly(ds)
    t_parts, res = [], np.zeros(3, dtype=int)
    for rank in range(world):
        a = _host_assembly(ds, shard=(rank, world))
        _assert_same_assembly(a, _host_assembly(_unsorted_copy(ds), shard=(rank, world)))
        assert np.array_equal(a["cells"], calc_times_cells(ds, a["used"][0]))
        t_parts.append(a["used"][0]); res += np.array(a["res"])
    assert np.array_equal(np.concatenate(t_parts), full["used"][0])
    assert tuple(res) == full["res"]
