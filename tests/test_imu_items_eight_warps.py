"""IMU items of the persistent Jacobian kernel at eight warps per CTA, with their tensor-core accumulators in registers.

  * CPU: the streaming form of imu_accel_rows / imu_gyro_rows (icc_imu_rows.cuh), which writes the parked rows 1 and 2 entry by
    entry to a strided destination (the kernel's lane-private park), gives bit for bit the row 0, parked rows and residuals of the
    array form, on a fast spin, a vanishing increment and a padding lane (all-zero quaternion);
  * CPU: a host-only handle with BASELINE config 4 cuts the IMU stream into min(132 x 8, chunks) runs, and config 4 has enough
    chunks to stay on the persistent path;
  * GPU: cost, residuals, J^T r and J^T J against the oracle with the IMU items forced onto the persistent kernel, in runs that carry
    a tile between chunks, straddle two cells and re-stage, under every lockstep group count (each group on one named barrier) and
    with lockstep off."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from helpers import F_STAGE1
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "openimucameracalibrator_b200", "csrc")
DP = ctypes.POINTER(ctypes.c_double)
IMU_WARPS = 8                 # warps per CTA of the IMU items (eval_tmem_warps(true))
HOST_SMS = 132                # SM count a host-only handle assumes
F_GRAV1 = F_STAGE1 | capi.FLAG_GRAVITY_DIR
ACC_PARK, GYR_PARK = 43, 38

HARNESS = r'''
#include "icc_imu_rows.cuh"
using namespace icc;
// One sample through both forms.  knots: so3 6 x (x,y,z,w), r3 6 x 3, ba / bg 3 x 3; zero_q: the window's first knot is replaced by the
// all-zero quaternion after staging (the parked quaternion of a padding lane).  Streaming form: row 0 at stride ld, park at stride ldp,
// into buffers the caller pre-fills.  out_arr = [acc row0 (40) | acc park (43) | ra (3) | gyr row0 (24) | gyr park (38) | rg (3)].
extern "C" void hm_imu_stream(const double* so3, const double* r3, const double* ba, const double* bg, const double* u4, const double* Ma,
                              const double* Mg, const double* grav, const double* w5, const double* a_meas, const double* g_meas, int zero_q,
                              int ld, int ldp, double* out_arr, double* acc_row0, double* acc_pk, double* ra, double* gyr_row0, double* gyr_pk, double* rg) {
  static ImuWin W; ImuConst K;
  for (int i = 0; i < 5; ++i) stage_frame_increment(W.f, i, q4(so3[4 * i], so3[4 * i + 1], so3[4 * i + 2], so3[4 * i + 3]), q4(so3[4 * i + 4], so3[4 * i + 5], so3[4 * i + 6], so3[4 * i + 7]));
  W.f.q0 = zero_q ? q4(0, 0, 0, 0) : q4(so3[0], so3[1], so3[2], so3[3]);
  for (int j = 0; j < 6; ++j) W.f.p[j] = v3(r3[3 * j], r3[3 * j + 1], r3[3 * j + 2]);
  for (int j = 0; j < 3; ++j) { W.ba[j] = v3(ba[3 * j], ba[3 * j + 1], ba[3 * j + 2]); W.bg[j] = v3(bg[3 * j], bg[3 * j + 1], bg[3 * j + 2]); }
  for (int i = 0; i < 9; ++i) { K.Ma[i] = Ma[i]; K.Mg[i] = Mg[i]; }
  K.grav = v3(grav[0], grav[1], grav[2]); K.w_acc = w5[0]; K.w_gyr = w5[1]; K.idt2 = w5[3] * w5[3]; K.inv_so3_dt = w5[2];
  const V3 am = v3(a_meas[0], a_meas[1], a_meas[2]), gm = v3(g_meas[0], g_meas[1], g_meas[2]);
  double pa[ACC_PARK], rra[3], pg[GYR_PARK], rrg[3];
  imu_accel_rows(W, K, u4[0], u4[1], u4[2], am, out_arr, 1, pa, rra);
  for (int j = 0; j < ACC_PARK; ++j) out_arr[40 + j] = pa[j];
  for (int j = 0; j < 3; ++j) out_arr[83 + j] = rra[j];
  imu_gyro_rows(W, K, u4[0], u4[3], gm, out_arr + 86, 1, pg, rrg);
  for (int j = 0; j < GYR_PARK; ++j) out_arr[110 + j] = pg[j];
  for (int j = 0; j < 3; ++j) out_arr[148 + j] = rrg[j];
  imu_accel_rows(W, K, u4[0], u4[1], u4[2], am, acc_row0, ld, acc_pk, ldp, *reinterpret_cast<double(*)[3]>(ra));
  imu_gyro_rows(W, K, u4[0], u4[3], gm, gyr_row0, ld, gyr_pk, ldp, *reinterpret_cast<double(*)[3]>(rg));
}
// The parked accelerometer row k (1, 2) expanded into 40 tile entries, as accel_part does.
extern "C" void hm_accel_expand(const double* park, const double* w5, int k, double* row) {
  ImuConst K; K.w_acc = w5[0]; K.idt2 = w5[3] * w5[3];
  double so3[18];
  for (int c = 0; c < 18; ++c) so3[c] = park[18 * (k - 1) + c];
  imu_accel_row_expand(so3, q4(park[36], park[37], park[38], park[39]), park[39 + k], park[42], K, k, row, 1);
}
'''


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    d = tmp_path_factory.mktemp("imu_stream")
    src, out = d / "imu_stream.cu", d / "libimu_stream.so"
    src.write_text(HARNESS)
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", CSRC, "-o", str(out), str(src)])
    return ctypes.CDLL(str(out))


def _qexp(w):
    th = np.linalg.norm(w)
    if th == 0.0:
        return np.array([0.0, 0.0, 0.0, 1.0])
    return np.concatenate([np.sin(th / 2) * w / th, [np.cos(th / 2)]])


def _qmul(a, b):
    ax, ay, az, aw = a; bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _knots(rng, steps):
    """Six SO(3) knots whose five increments are the given rotation vectors."""
    q = [_qexp(rng.normal(0, 0.6, 3))]
    for w in steps:
        q.append(_qmul(q[-1], _qexp(np.asarray(w, dtype=np.float64))))
    return np.array(q)


def _cases():
    rng = np.random.default_rng(5)
    fast = [rng.normal(0, 1.0, 3) / np.sqrt(3) * a for a in (2.8, 2.0, 1.2, 2.5, 0.9)]     # half-angles beyond pi/4: library sincos
    still = [np.zeros(3), rng.normal(0, 1e-3, 3), np.zeros(3), np.zeros(3), rng.normal(0, 1e-3, 3)]
    mild = [rng.normal(0, 0.1, 3) for _ in range(5)]
    return [("fast_spin", _knots(rng, fast), False), ("vanishing_increment", _knots(rng, still), False), ("padding_lane", _knots(rng, mild), True)]


def _run(hs, so3, zero_q, ld, ldp, rng):
    r3 = rng.normal(0, 0.5, (6, 3)); ba = rng.normal(0, 0.05, (3, 3)); bg = rng.normal(0, 0.01, (3, 3))
    u4 = rng.uniform(0.02, 0.97, 4)
    Ma = np.array([[1.01, -0.002, 0.003], [0, 0.99, -0.001], [0, 0, 1.02]]); Mg = np.eye(3) + rng.normal(0, 0.003, (3, 3))
    grav = np.array([0.1, -0.2, 9.8]); w5 = np.array([3.0, 40.0, 20.0, 20.0])      # w_acc, w_gyr, inv_so3_dt, inv_r3_dt
    a_meas, g_meas = rng.normal(0, 3, 3), rng.normal(0, 1, 3)
    arr = np.zeros(151)
    bufs = {"acc_row0": np.full(40 * ld, np.nan), "acc_pk": np.full(ACC_PARK * ldp, np.nan), "ra": np.zeros(3),
            "gyr_row0": np.full(24 * ld, np.nan), "gyr_pk": np.full(ACC_PARK * ldp, np.nan), "rg": np.zeros(3)}
    ins = [np.ascontiguousarray(x, dtype=np.float64) for x in (so3, r3, ba, bg, u4, Ma, Mg, grav, w5, a_meas, g_meas)]
    hs.hm_imu_stream(*[x.ctypes.data_as(DP) for x in ins], ctypes.c_int(int(zero_q)), ctypes.c_int(ld), ctypes.c_int(ldp), arr.ctypes.data_as(DP),
                     *[bufs[k].ctypes.data_as(DP) for k in ("acc_row0", "acc_pk", "ra", "gyr_row0", "gyr_pk", "rg")])
    return arr, bufs, w5


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, dtype=np.float64).view(np.uint64), np.ascontiguousarray(b, dtype=np.float64).view(np.uint64))


@pytest.mark.parametrize("case", ["fast_spin", "vanishing_increment", "padding_lane"])
def test_streaming_rows_equal_the_array_form_bit_for_bit(hs, case):
    name, so3, zero_q = next(c for c in _cases() if c[0] == case)
    rng = np.random.default_rng(11)
    ld, ldp = 3, 5
    arr, b, w5 = _run(hs, so3, zero_q, ld, ldp, rng)
    assert np.all(np.isfinite(arr)), name
    assert _same_bits(b["acc_row0"][::ld], arr[:40]) and _same_bits(b["acc_pk"][::ldp], arr[40:83]) and _same_bits(b["ra"], arr[83:86]), name
    assert _same_bits(b["gyr_row0"][::ld], arr[86:110]) and _same_bits(b["gyr_pk"][: GYR_PARK * ldp : ldp], arr[110:148]) and _same_bits(b["rg"], arr[148:151]), name
    # nothing is written between the strided entries, nor past the gyroscope's 38 parked doubles
    for k in ("acc_row0", "gyr_row0"):
        assert np.all(np.isnan(b[k].reshape(-1, ld)[:, 1:])), (name, k)
    for k, n in (("acc_pk", ACC_PARK), ("gyr_pk", GYR_PARK)):
        assert np.all(np.isnan(b[k].reshape(-1, ldp)[:, 1:])) and np.all(np.isnan(b[k][n * ldp:])), (name, k)
    if zero_q:                            # the parked quaternion marks the lane as padding: its expanded rows are zero but for the residual
        assert not np.any(arr[76:80])
        for k in (1, 2):
            row = np.zeros(40)
            hs.hm_accel_expand(arr[40:83].ctypes.data_as(DP), w5.ctypes.data_as(DP), ctypes.c_int(k), row.ctypes.data_as(DP))
            assert not np.any(row[18:39]) and row[39] == arr[79 + k], k


def test_config4_imu_runs_fill_eight_warps_per_sm(monkeypatch):
    """The schedule is host logic: a host-only handle (132 SMs) gives BASELINE config 4 min(132 x 8, chunks) IMU runs, and enough
    chunks that the size test of launch_eval keeps its IMU items on the persistent kernel."""
    from openimucameracalibrator_b200 import calibrator
    monkeypatch.delenv("ICC_TMEM_RUNS", raising=False)
    h = capi.CApi(calibrator.load_library(), "icc_", -1)
    capi.load_dataset(h, syn.make_dataset(syn.CONFIGS[4]))
    s = h.eval_schedule()
    h.close()
    warps = HOST_SMS * IMU_WARPS
    assert len(s["iitems"]) == min(warps, s["n_ichunks"])
    assert 2 * s["n_ichunks"] >= 3 * warps, s["n_ichunks"]
    assert len(s["vitems"]) == min(warps, s["n_vchunks"])


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
LOCKSTEP = [("groups", "1"), ("groups", "2"), ("groups", "4"), ("groups", "8"), ("no_lockstep", "1")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,value", LOCKSTEP)
def test_imu_items_with_free_gravity_under_every_lockstep_group(oracle_factory, gpu_factory, monkeypatch, mode, value):
    from test_gpu_parity import _assert_eval_parity
    from test_gpu_tmem_runs import checked_schedule
    monkeypatch.setenv("ICC_TMEM_ALWAYS", "1")
    monkeypatch.delenv("ICC_TMEM_STAGGER_NS", raising=False)
    if mode == "groups":
        monkeypatch.setenv("ICC_TMEM_GROUPS", value); monkeypatch.delenv("ICC_TMEM_NO_LOCKSTEP", raising=False)
    else:
        monkeypatch.setenv("ICC_TMEM_NO_LOCKSTEP", value); monkeypatch.delenv("ICC_TMEM_GROUPS", raising=False)
    ds = syn.make_dataset(syn.tiny_config(n_frames=20, imu_rate_hz=1000.0))
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    seen = set()
    for cap in (1, 7, 13, None):
        if cap is None:
            monkeypatch.delenv("ICC_TMEM_RUNS", raising=False)
        else:
            monkeypatch.setenv("ICC_TMEM_RUNS", str(cap))
        g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
        seen |= checked_schedule(g, ds, cap)["imu"]
        _assert_eval_parity(o, g, F_GRAV1)
        g.close()
    o.close()
    assert {"carry", "straddle", "restage"} <= seen, seen
