"""Multi-chunk runs of the persistent Jacobian kernel (icc_eval_tmem.cu) against the CPU oracle.

batch_init cuts each packed stream (corners of the non-empty frames, samples of the IMU cells, units padded to a multiple of 4) into
at most sm_count x 6 per-warp runs.  A warp carries tile state from one chunk to the next only when its run has several chunks:
accumulators parked while a frame / cell spans chunks, the two staged windows swapped after a chunk that straddles two units, the
re-stage when a unit ends exactly on a chunk boundary, runs that start or end inside a unit, and the trailing lockstep barriers of
runs shorter than the longest.  The small parity cases give every warp one chunk, so ICC_TMEM_RUNS=n (read by batch_init) caps the
run count here to put every one of those states on the path, and icc_get_eval_schedule shows which ones a case contains.

  * CPU: a NumPy statement of the host walk + split and of the kernel's run loop, checked for consistency on ragged unit sizes; the
    library's schedule, which batch_init computes on a host-only handle too, equals the statement;
  * GPU: the same on GPU handles; cost, residuals, J^T r and J^T J agree with the oracle for every camera model
    and the column sets of both stages -- including SPLINE | T_I_C | GRAVITY_DIR, the hot CLI's stage 1 with unknown gravity, whose
    gravity columns only the persistent IMU items carry -- on ragged frames, irregular IMU streams and at config-2 size."""
import numpy as np
import pytest

from helpers import F_ALL, F_STAGE1, F_STAGE2, rel
from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import synthetic as syn
from scaled_parity import assert_block_probes, probe_reference

CHUNK = 32
CTA_WARPS = 6                   # warps per CTA of the persistent kernel (eval_tmem_warps)
F_GRAV1 = F_STAGE1 | capi.FLAG_GRAVITY_DIR


# ---- NumPy statement of the schedule ---------------------------------------------------------------------------------------------
def padded_offsets(sizes):
    """Packed-stream offsets of the units (each padded to a multiple of 4) plus the two sentinels the kernel reads past the end."""
    sizes = np.asarray(sizes, dtype=np.int64)
    assert np.all(sizes > 0)
    poff = np.concatenate([[0], np.cumsum((sizes + 3) // 4 * 4)])
    return [int(x) for x in poff] + [int(poff[-1])]


def walk(poff):
    """Host walk (icc_api.cu, batch_init): chunks of up to 32 positions from at most two consecutive units -> [(pos, unit)]."""
    n_units, total = len(poff) - 2, poff[-1]
    chunks, pos, u = [], 0, 0
    while pos < total:
        while poff[u + 1] <= pos:
            u += 1
        chunks.append((pos, u))
        n_a = min(CHUNK, poff[u + 1] - pos)
        n = n_a
        if n_a < CHUNK and u + 1 < n_units:
            n += min(CHUNK - n_a, poff[u + 2] - poff[u + 1])
        pos += n
    return chunks


def split(chunks, total, cap):
    """Even runs, one per warp: at most `cap` runs -> [(first unit, pos_begin, pos_end)]."""
    nc = len(chunks)
    n_items = min(cap, nc)
    items = []
    for k in range(n_items):
        a, b = nc * k // n_items, nc * (k + 1) // n_items
        items.append((chunks[a][1], chunks[a][0], chunks[b][0] if b < nc else total))
    return items


def schedule(sizes, cap):
    poff = padded_offsets(sizes) if len(sizes) else [0, 0, 0]
    chunks = walk(poff)
    return poff, chunks, split(chunks, poff[-1], cap)


def run_loop(poff, item):
    """The kernel's loop over one run (tmv::run_item / tmi::run_item): one record per chunk with its tile parts
    (unit, k0, k1, first, last) -- first: accumulators start at zero (else fetched from the park); last: scattered (else parked)."""
    f, pos, pos_end = item
    end_f = min(poff[f + 1], pos_end)
    fresh, out = True, []
    while pos < pos_end:
        restage = pos == end_f
        if restage:                                   # the previous chunk finished its unit exactly at the chunk boundary
            f += 1
            end_f = min(poff[f + 1], pos_end)
            fresh = True
        n_a = min(CHUNK, end_f - pos)
        n_b, end_b = 0, 0
        if n_a < CHUNK and end_f < pos_end:           # the unit ends inside this chunk: the remaining lanes start the next one
            assert f + 2 < len(poff)                  # (reads stay within the two sentinels)
            end_b = min(poff[f + 2], pos_end)
            n_b = min(CHUNK - n_a, end_b - end_f)
        n = n_a + n_b
        assert n_a % 4 == 0 and n_b % 4 == 0 and n > 0
        parts = [(f, 0, n_a >> 2, fresh, pos + n_a == end_f)]
        if n_b:
            parts.append((f + 1, n_a >> 2, n >> 2, True, end_f + n_b == end_b))
        out.append(dict(pos=pos, n=n, unit=f, parts=parts, restage=restage, straddle=n_b > 0))
        fresh = False
        if n_b:
            f += 1
            end_f = end_b
        pos += n
    return out


def check_schedule(poff, chunks, items):
    """Every run's loop visits exactly the chunks the walk counted for it, no run exceeds the lockstep rounds, the runs tile the
    stream once, and every parked accumulator is fetched by the very next tile part of the same unit (one park per warp)."""
    total, nc = poff[-1], len(chunks)
    if nc == 0:
        assert items == []
        return
    rounds = -(-nc // len(items))
    assert items[0][1] == 0 and items[-1][2] == total
    seen = np.zeros(total, dtype=np.int32)
    k = 0
    for it in items:
        loop = run_loop(poff, it)
        assert len(loop) <= rounds
        assert [(c["pos"], c["unit"]) for c in loop] == chunks[k: k + len(loop)]
        k += len(loop)
        assert loop[-1]["pos"] + loop[-1]["n"] == it[2]
        parked = None
        for c in loop:
            for unit, k0, k1, first, last in c["parts"]:
                assert first == (parked is None) and (first or parked == unit)
                assert poff[unit] <= c["pos"] + 4 * k0 and c["pos"] + 4 * k1 <= poff[unit + 1]
                parked = None if last else unit
                seen[c["pos"] + 4 * k0: c["pos"] + 4 * k1] += 1
        assert parked is None                         # every run scatters what it accumulated
    assert k == nc
    assert np.all(seen == 1)
    for a, b in zip(items, items[1:]):
        assert a[2] == b[1]


def run_features(poff, items):
    """Which carry states a stream's runs put on the path."""
    if not items:
        return set()
    loops = [run_loop(poff, it) for it in items]
    lengths = [len(x) for x in loops]
    feats = set()
    if any(not p[3] for x in loops for c in x for p in c["parts"]):
        feats.add("carry")                            # accumulators fetched from the park
    if any(c["straddle"] for x in loops for c in x):
        feats.add("straddle")
    if any(c["restage"] for x in loops for c in x):
        feats.add("restage")                          # a unit ended exactly on a chunk boundary inside a run
    if any(it[1] != poff[it[0]] for it in items):
        feats.add("mid_start")
    if any(it[2] not in poff for it in items):
        feats.add("mid_end")
    if min(lengths) != max(lengths):
        feats.add("uneven")                           # shorter runs finish with trailing lockstep barriers
    if len(items) % CTA_WARPS:
        feats.add("idle_warps")                       # the grid's last warps have no run
    return feats


RAGGED = [1, 2, 3, 4, 5, 31, 32, 33, 36, 63, 64, 65, 1, 3, 2, 1, 3, 96, 7, 144, 50, 50, 8, 2, 2, 2, 29, 100]
CAPS = [1, 5, 6, 7, 13, 10_000]


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("seed", [None, 0, 1, 2])
def test_schedule_statement_is_consistent(cap, seed):
    sizes = RAGGED if seed is None else list(np.random.default_rng(seed).integers(1, 120, size=60))
    poff, chunks, items = schedule(sizes, cap)
    assert len(items) == min(cap, len(chunks))
    check_schedule(poff, chunks, items)
    if cap in (1, 5, 7) and seed is None:
        assert {"carry", "straddle", "restage"} <= run_features(poff, items)
        assert cap == 1 or {"mid_start", "mid_end"} <= run_features(poff, items)


def test_schedule_statement_edges():
    for sizes in ([], [1], [4], [32], [33], [64], [1] * 40, [3, 29], [30, 2, 32], [28, 4, 32, 1]):
        for cap in CAPS:
            poff, chunks, items = schedule(sizes, cap)
            check_schedule(poff, chunks, items)
    # one 32-corner unit per chunk: no straddle, and every unit boundary inside a run is a re-stage
    assert run_features(*schedule([32] * 10, 3)[::2]) >= {"restage", "uneven"}
    assert "straddle" not in run_features(*schedule([32] * 10, 3)[::2])
    assert run_features(*schedule([40, 40], 1)[::2]) >= {"carry", "straddle"}


def test_features_name_what_they_see():
    poff, _, items = schedule([96] * 5, 1)            # one run, frames of exactly 3 chunks
    assert run_features(poff, items) == {"carry", "restage", "idle_warps"}
    poff, _, items = schedule([96] * 4, 6)            # 12 chunks, 6 runs of 2: frames start and end inside runs
    assert run_features(poff, items) == {"carry", "restage", "mid_start", "mid_end"}
    poff, _, items = schedule([96] * 4, 5)            # 12 chunks in runs of 2 or 3
    assert {"uneven", "idle_warps"} <= run_features(poff, items)


def test_schedule_getter_needs_an_assembled_problem():
    from openimucameracalibrator_b200 import calibrator
    h = capi.CApi(calibrator.load_library(), "icc_", -1)             # host-only handle
    with pytest.raises(capi.IccError, match="ICC_ERR_STATE"):
        h.eval_schedule()
    h.close()


# ---- GPU: the library's schedule and its evaluations ------------------------------------------------------------------------------
@pytest.fixture()
def tmem_runs(monkeypatch):
    """Forces the persistent kernel (ICC_TMEM_ALWAYS) and caps its runs (ICC_TMEM_RUNS; None = the default sm_count x 6)
    for the handles loaded after the call."""
    def set_cap(cap):
        monkeypatch.setenv("ICC_TMEM_ALWAYS", "1")
        if cap is None:
            monkeypatch.delenv("ICC_TMEM_RUNS", raising=False)
        else:
            monkeypatch.setenv("ICC_TMEM_RUNS", str(cap))
    return set_cap


def stream_units(g, ds):
    """Unit sizes of the two packed streams of a loaded handle: the corner counts of the non-empty frames (every frame of these
    datasets is kept) and the sample counts of the IMU cells."""
    counts = np.diff(ds["corner_offsets"])
    assert g.num_residuals()[0] == 2 * int(counts.sum())
    cells = g.imu_cells()
    return [int(c) for c in counts if c > 0], [int(c) for c in cells[:, 5] - cells[:, 4] if c > 0]


def checked_schedule(g, ds, cap):
    """The library's schedule must equal the NumPy statement exactly; returns the features of both streams."""
    s = g.eval_schedule()
    feats = {}
    for name, sizes, n_chunks, items in zip(("vision", "imu"), stream_units(g, ds), (s["n_vchunks"], s["n_ichunks"]), (s["vitems"], s["iitems"])):
        got = [tuple(int(x) for x in r) for r in items]
        if cap is None:                               # default: min(sm_count x 6, chunks) runs
            assert len(got) == n_chunks or len(got) % CTA_WARPS == 0, name
        poff, chunks, want = schedule(sizes, cap if cap is not None else max(len(got), 1))
        assert n_chunks == len(chunks), name
        assert got == want, name
        check_schedule(poff, chunks, want)
        feats[name] = run_features(poff, want)
    return feats


class CachedOracle:
    """The oracle's evaluations do not depend on the GPU's schedule: evaluate each column set once."""

    def __init__(self, o):
        self.o, self.memo = o, {}

    def evaluate(self, flags, **kw):
        key = (flags, tuple(sorted(kw.items())))
        if key not in self.memo:
            self.memo[key] = self.o.evaluate(flags, **kw)
        return self.memo[key]


def _parity(oracle_factory, gpu_factory, tmem_runs, ds, caps, flag_sets, **kw):
    """Every column set under every cap against the oracle; each schedule must carry a tile between chunks and straddle two units.
    Returns the features each stream showed under any of the caps."""
    from test_gpu_parity import _assert_eval_parity
    o = oracle_factory(); capi.load_dataset(o, ds, **kw)
    oc = CachedOracle(o)
    seen = {"vision": set(), "imu": set()}
    for cap in caps:
        tmem_runs(cap)
        g = gpu_factory(); capi.load_dataset(g, ds, **kw)
        feats = checked_schedule(g, ds, cap)
        assert {"carry", "straddle"} <= feats["vision"] | feats["imu"], (cap, feats)
        for flags in flag_sets:
            _assert_eval_parity(oc, g, flags)
        for s in seen:
            seen[s] |= feats[s]
        g.close()
    o.close()
    return seen


MATRIX_FLAGS = (F_STAGE1, F_GRAV1, capi.FLAG_SPLINE | capi.FLAG_GRAVITY_DIR, F_STAGE2, F_ALL, capi.FLAG_T_I_C)


SCHEDULE_CAPS = (None, 1, 5, 6, 7, 13, 96)


def _schedule_cases():
    return [syn.make_dataset(syn.tiny_config(n_frames=30, dt_so3_s=0.04, dt_r3_s=0.07)), syn.make_dataset(syn.tiny_config(imu_rate_hz=1000.0, n_frames=20)),
            _ragged_dataset()]


def test_host_only_schedule_matches_the_statement(tmem_runs):
    """The schedule is host logic: a host-only handle (whose default run count assumes 132 SMs) computes it without a GPU."""
    from openimucameracalibrator_b200 import calibrator
    for ds in _schedule_cases():
        for cap in SCHEDULE_CAPS:
            tmem_runs(cap)
            h = capi.CApi(calibrator.load_library(), "icc_", -1); capi.load_dataset(h, ds)
            checked_schedule(h, ds, cap)
            h.close()


@pytest.mark.gpu
def test_schedule_matches_the_statement(gpu_factory, tmem_runs):
    for ds in _schedule_cases():
        for cap in SCHEDULE_CAPS:
            tmem_runs(cap)
            g = gpu_factory(); capi.load_dataset(g, ds)
            checked_schedule(g, ds, cap)
            g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(8))
def test_every_model_and_column_set_in_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs, k):
    cfg = syn.config5(k); cfg.n_frames = 20
    _parity(oracle_factory, gpu_factory, tmem_runs, syn.make_dataset(cfg), (1, 7, 13), MATRIX_FLAGS, known_gravity=False)


@pytest.mark.gpu
def test_pinhole_radial_tangential_in_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs):
    cfg = syn.tiny_config(cm.PINHOLE_RADIAL_TANGENTIAL, (440.0, 1.01, 0.2, 480.0, 270.0, -0.1, 0.02, -0.003, 1e-3, -2e-3), seed=3)
    _parity(oracle_factory, gpu_factory, tmem_runs, syn.make_dataset(cfg), (1, 7, 13), MATRIX_FLAGS, known_gravity=False)


RAGGED_FRAMES = [0, 1, 2, 3, 4, 5, 31, 32, 33, 36, 63, 64, 65, 1, 3, 2, 1, 2, 3, 65, 0, 64, 33, 5]


def _ragged_dataset():
    """Frames of 0..65 corners, including a run of consecutive 1-3-corner frames; shuffled corner subsets of a 13 x 5 board."""
    ds = dict(syn.make_dataset(syn.tiny_config(grid=(13, 5), n_frames=len(RAGGED_FRAMES), seed=17)))
    C = 65
    rng = np.random.default_rng(4)
    off, ids, uv = [0], [], []
    for f, n in enumerate(RAGGED_FRAMES):
        sel = np.sort(rng.choice(C, size=n, replace=False))
        ids.append(ds["point_ids"][f * C + sel]); uv.append(ds["uv"][f * C + sel]); off.append(off[-1] + n)
    ds["corner_offsets"] = np.array(off, dtype=np.int32); ds["point_ids"] = np.concatenate(ids).astype(np.int32); ds["uv"] = np.concatenate(uv)
    return ds


@pytest.mark.gpu
def test_ragged_frames_in_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs):
    seen = _parity(oracle_factory, gpu_factory, tmem_runs, _ragged_dataset(), (1, 5, 7), (F_ALL, F_GRAV1, F_STAGE2), known_gravity=False)
    assert seen["vision"] >= {"carry", "straddle", "restage", "mid_start", "mid_end", "uneven", "idle_warps"}, seen


def _irregular_stamps_dataset():
    """IMU stamps on knot boundaries of both grids, repeated stamps and an irregular rate, dt_so3 != dt_r3."""
    ds = dict(syn.make_dataset(syn.tiny_config(n_frames=30, dt_so3_s=0.04, dt_r3_s=0.07)))
    rng = np.random.default_rng(12)
    t0 = float(ds["frame_t"][0]) - ds["time_offset_imu_to_cam_s"]
    n = len(ds["imu_t"])
    t = np.sort(rng.uniform(ds["imu_t"][0], ds["imu_t"][-1], size=n))
    k = np.arange(0, n, 7)
    t[k] = t0 + 0.04 * np.round((t[k] - t0) / 0.04)
    k = np.arange(3, n, 11)
    t[k] = t0 + 0.07 * np.round((t[k] - t0) / 0.07)
    t = np.sort(t); t[5::13] = t[4::13][: len(t[5::13])]
    ds["imu_t"] = np.sort(t)
    return ds


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["stamps", "low_rate", "1khz"])
def test_imu_edges_with_free_gravity_in_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs, case):
    if case == "stamps":
        ds = _irregular_stamps_dataset()
    elif case == "low_rate":
        ds = syn.make_dataset(syn.tiny_config(n_frames=30, imu_rate_hz=50.0, dt_so3_s=0.04, dt_r3_s=0.07))
    else:
        ds = syn.make_dataset(syn.tiny_config(n_frames=20, imu_rate_hz=1000.0))
    _parity(oracle_factory, gpu_factory, tmem_runs, ds, (1, 7), (F_GRAV1,), known_gravity=False)
    tmem_runs(7)
    g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
    sizes = stream_units(g, ds)[1]
    if case == "low_rate":
        assert 1 <= min(sizes) and max(sizes) <= 3
    elif case == "1khz":
        assert max(sizes) > CHUNK and "carry" in checked_schedule(g, ds, 7)["imu"]


@pytest.mark.gpu
def test_config2_schedule_invariance(oracle_factory, gpu_factory, tmem_runs):
    """At config-2 size the default schedule (one or two chunks per warp on a 132-SM H100) and capped ones agree with the oracle."""
    ds = syn.make_dataset(syn.CONFIGS[2])
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    rng = np.random.default_rng(44)
    ref = {}
    for flags in (F_STAGE1, F_GRAV1):
        co, _, go, _ = o.evaluate(flags, residuals=False)
        n = o.num_tangent(flags)
        V = rng.normal(size=(4, n)); V[1, : n - 9] = 0.0; V[2, n - 9:] = 0.0      # all columns / border only / band only / all
        ref[flags] = (co, go, V, o.normal_matvec(flags, V))
    probes = {flags: probe_reference(o, flags, rng) for flags in ref}           # each column block and the end knots at their own scale
    for cap in (None, 96, 7):
        tmem_runs(cap)
        g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
        feats = checked_schedule(g, ds, cap)
        if cap is not None:                           # (config 2's 10-sample cells never span chunks: its IMU runs re-stage instead)
            assert "carry" in feats["vision"] and "restage" in feats["imu"], (cap, feats)
        for flags, (co, go, V, Ho) in ref.items():
            cg, _, gg, _ = g.evaluate(flags, residuals=False)
            assert abs(cg - co) <= 1e-9 * co and rel(gg, go) < 1e-9, (cap, flags)
            for a, b in zip(g.normal_matvec(flags, V), Ho):
                assert rel(a, b) < 1e-9, (cap, flags)
            assert_block_probes(g, probes[flags])
        g.close()


@pytest.mark.gpu
def test_config1_lm_with_free_gravity(oracle_factory, gpu_factory, tmem_runs):
    ds = syn.make_dataset(syn.CONFIGS[1])
    o = oracle_factory(); capi.load_dataset(o, ds, known_gravity=False)
    so = o.optimize(50, F_GRAV1)
    for cap in (7, None):
        tmem_runs(cap)
        g = gpu_factory(); capi.load_dataset(g, ds, known_gravity=False)
        sg = g.optimize(50, F_GRAV1)
        assert sg.iterations == so.iterations and sg.termination == so.termination, cap
        assert rel(g.get_T_i_c(), o.get_T_i_c()) < 1e-8 and rel(g.get_gravity(), o.get_gravity()) < 1e-8, cap
        g.close()


@pytest.mark.gpu
def test_points_in_multi_chunk_runs(oracle_factory, gpu_factory, tmem_runs):
    flags = F_STAGE1 | capi.FLAG_POINTS
    ds = syn.make_dataset(syn.tiny_config(model=cm.DOUBLE_SPHERE, intr=(342.4, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513), n_frames=16))
    tmem_runs(7)
    g = gpu_factory(); capi.load_dataset(g, ds)
    o = oracle_factory(); capi.load_dataset(o, ds)
    assert {"carry", "straddle"} <= checked_schedule(g, ds, 7)["vision"]
    npts = len(ds["board_xyzw"])
    n = g.num_tangent(flags)
    assert n == o.num_tangent(flags) == g.num_tangent(F_STAGE1) + 3 * npts
    cg, rg, gg, _ = g.evaluate(flags)
    co, ro, go, _ = o.evaluate(flags)
    assert abs(cg - co) <= 1e-11 * co and rel(rg, ro) < 1e-9
    assert rel(gg, go) < 1e-9 and rel(gg[n - 3 * npts:], go[n - 3 * npts:]) < 1e-9
    rng = np.random.default_rng(8)
    V = rng.normal(size=(4, n)); V[1, : n - 3 * npts] = 0.0; V[2, n - 3 * npts:] = 0.0
    for a, b in zip(g.normal_matvec(flags, V), o.normal_matvec(flags, V)):
        assert rel(a, b) < 1e-9
    assert_block_probes(g, probe_reference(o, flags, rng))
