"""The SO(3) increment table of the persistent Jacobian kernel (incr_table_entry, icc_vision_rows.cuh; incr_table_kernel,
icc_eval_tmem.cu): every knot increment's log, unit axis, norm and Jr^-1 formed once per evaluation, and knot windows staged by copying
five entries out of it instead of recomputing them.

  * CPU: a window assembled from table entries (incr_table_index, the copy the staging functions make) is bit-identical to
    stage_frame_increment on the same knots, for every window of knot sequences with a fast spin, vanishing increments (0, 1e-12,
    1e-8 rad) and increments up to 2.8 rad, including the first and the last window of the sequence;
  * GPU: the table is rebuilt from the state each evaluation runs on: after set_knots moves the knots between two evaluations of
    BASELINE config 4, the second evaluation's cost, J^T r and J^T J agree with the oracle at the new knots."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from helpers import F_STAGE1, qexp, qmul, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_block_probes, probe_reference

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "openimucameracalibrator_b200", "csrc")
DP = ctypes.POINTER(ctypes.c_double)
IP = ctypes.POINTER(ctypes.c_int)
WIN_INCR = 85                 # doubles of a window's increment block (FrameWin::d .. FrameWin::jri)

HARNESS = r'''
#include <cstring>
#include <vector>
#include "icc_vision_rows.cuh"
using namespace icc;
// knots: n_so3 x (x,y,z,w).  For window k starting at knot starts[k]: the increment block assembled from the table into
// from_table[85 k ..] and the one stage_frame_increment stages into staged[85 k ..].
extern "C" void hm_incr_windows(const double* knots, int n_so3, const int* starts, int n_starts, double* from_table, double* staged) {
  const int n = n_so3 - 1;
  std::vector<double4> q(n_so3);
  for (int i = 0; i < n_so3; ++i) q[i] = make_double4(knots[4 * i], knots[4 * i + 1], knots[4 * i + 2], knots[4 * i + 3]);
  std::vector<double> tab((size_t)INCR_DOUBLES * n);
  for (int i = 0; i < n; ++i) incr_table_entry(q.data(), i, n, tab.data());
  for (int k = 0; k < n_starts; ++k) {
    const int s = starts[k];
    static FrameWin A, B;
    memset(&A, 0, sizeof A); memset(&B, 0, sizeof B);
    double* a = win_incr(A);
    for (int e = 0; e < WIN_INCR_DOUBLES; ++e) a[e] = tab[incr_table_index(e, s, n)];
    for (int i = 0; i < 5; ++i)
      stage_frame_increment(B, i, q4(q[s + i].x, q[s + i].y, q[s + i].z, q[s + i].w), q4(q[s + i + 1].x, q[s + i + 1].y, q[s + i + 1].z, q[s + i + 1].w));
    memcpy(from_table + (size_t)WIN_INCR_DOUBLES * k, win_incr(A), WIN_INCR_DOUBLES * sizeof(double));
    memcpy(staged + (size_t)WIN_INCR_DOUBLES * k, win_incr(B), WIN_INCR_DOUBLES * sizeof(double));
  }
}
'''


@pytest.fixture(scope="module")
def hm(tmp_path_factory):
    d = tmp_path_factory.mktemp("incr_table")
    src, out = d / "incr_table.cu", d / "libincr_table.so"
    src.write_text(HARNESS)
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-I", CSRC, "-o", str(out), str(src)])
    return ctypes.CDLL(str(out))


def knots_from_increments(angles, rng):
    """Knot sequence whose consecutive increments have the given angles about random unit axes."""
    q = [qexp(rng.normal(size=3))]
    for a in angles:
        ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
        q.append(qmul(q[-1], qexp(a * ax)))
    return np.array(q)


def windows(hm, knots):
    n_so3 = len(knots)
    starts = np.arange(n_so3 - 5, dtype=np.int32)            # every window, the first and the last included
    a, b = np.zeros((len(starts), WIN_INCR)), np.zeros((len(starts), WIN_INCR))
    k = np.ascontiguousarray(knots, dtype=np.float64)
    hm.hm_incr_windows(k.ctypes.data_as(DP), n_so3, starts.ctypes.data_as(IP), len(starts), a.ctypes.data_as(DP), b.ctypes.data_as(DP))
    return a, b


@pytest.mark.parametrize("case", ["fast_spin", "vanishing", "large", "mixed"])
def test_window_from_table_is_bit_identical_to_staging(hm, case):
    rng = np.random.default_rng(7)
    if case == "fast_spin":                                   # 48 rad/s at 0.05 s knot spacing
        angles = np.full(30, 2.4)
    elif case == "vanishing":
        angles = np.array([0.0, 1e-12, 1e-8, 0.0, 0.0, 1e-12, 1e-8, 1e-8, 0.0, 1e-12, 0.0, 0.0])
    elif case == "large":
        angles = np.linspace(1.5, 2.8, 20)
    else:
        angles = np.concatenate([[0.0, 1e-12, 1e-8], rng.uniform(0.0, 2.8, 25), [1e-8, 0.0, 2.8]])
    knots = knots_from_increments(angles, rng)
    a, b = windows(hm, knots)
    assert a.view(np.int64).tobytes() == b.view(np.int64).tobytes()
    th = a[:, 30:35]                                          # the staged norms are the increments' angles
    assert np.allclose(th[:, 0], angles[: len(th)], atol=1e-9)
    assert np.allclose(th[-1], angles[-5:], atol=1e-9)


@pytest.mark.gpu
def test_table_follows_set_knots(oracle_factory, gpu_factory, monkeypatch):
    monkeypatch.setenv("ICC_TMEM_ALWAYS", "1")
    ds = syn.make_dataset(syn.CONFIGS[4])
    g = gpu_factory(); capi.load_dataset(g, ds)
    o = oracle_factory(); capi.load_dataset(o, ds)
    g.evaluate(F_STAGE1, residuals=False)                     # a table from the initial knots
    so3 = g.get_knots()[0]
    rng = np.random.default_rng(12)
    moved = np.array([qmul(q, qexp(rng.normal(scale=0.02, size=3))) for q in so3])
    g.set_knots(so3=moved); o.set_knots(so3=moved)
    cg, _, gg, _ = g.evaluate(F_STAGE1, residuals=False)
    co, _, go, _ = o.evaluate(F_STAGE1, residuals=False)
    assert abs(cg - co) <= 1e-10 * co
    assert rel(gg, go) < 1e-9
    n = g.num_tangent(F_STAGE1)
    V = rng.normal(size=(2, n)); V[1, : n - 6] = 0.0
    for a, b in zip(g.normal_matvec(F_STAGE1, V), o.normal_matvec(F_STAGE1, V)):
        assert rel(a, b) < 1e-9
    assert_block_probes(g, probe_reference(o, F_STAGE1, rng))
