"""The IMU-to-camera rotation initialiser (row f3) on streams that wake the code test_rotation_init.py leaves idle: mountings whose
rotation has trace <= 0 (the three other branches of the matrix-to-quaternion rule), q / -q flips between views and spin bursts past
2 pi rad/s (the outlier hold, including its "zero for i <= 1" rule), gyroscope spikes (the Huber branch of the error), permuted,
reversed and duplicated input, an irregular gyroscope clock with a gap, and windows of 12, 257 and 239800 samples (the last one past
the 4 x 132 x 256 = 135168 threads of one grid-stride pass of the sums and error reductions on an H100).

Every case runs the analytic scene of test_rotation_init.py.  GPU (-m gpu): the CUDA path reproduces the oracle with the parity bars
of test_rotation_init.py.  CPU: the oracle lands on the truth where the reference's estimator can; a NumPy restatement of the
front end (applications/estimate_imu_to_camera_rotation.cc:96-162, imu_to_camera_rotation_estimator.cc:116-215) shows that each input
really reaches the branch it is meant for.

Where the reference's estimator cannot recover the truth, only parity is asserted: a q / -q flip turns one finite difference into the
negated rate (the vector part of (-q_{i+1} - q_i) q_i^-1 is minus that of (q_{i+1} - q_i) q_i^-1), which no outlier test catches; held or spiked samples bias the closed-form rotation, which is not robust (only the error is); a reversed gyroscope file
gives a negative IMU period (taken in file order, as the reference does), which negates every visual rate; and 12 or 257 samples, an
irregular clock with a gap, or a 1 kHz gyroscope do not determine the offset to the reference's accuracy."""
import numpy as np
import pytest

from test_rotation_init import CONJ, Q_IC, _analytic, _qdiff, _rot

BIAS = np.array([0.004, -0.002, 0.001])
TD = 0.1
GRID_CAP = 4 * 132 * 256


def _mount(rotvec):
    v = np.asarray(rotvec, dtype=np.float64); th = np.linalg.norm(v)
    return np.r_[np.sin(th / 2) * v / th, np.cos(th / 2)] if th > 0 else np.array([0.0, 0.0, 0.0, 1.0])


_AX = np.random.default_rng(5).normal(size=3)
MOUNTINGS = {"x180": _mount([np.pi, 0, 0]), "y180": _mount([0, np.pi, 0]), "z180": _mount([0, 0, np.pi]), "identity": _mount([0, 0, 0]),
             "random": _mount(2.4 * _AX / np.linalg.norm(_AX))}


def _qmat(q):                                           # (x, y, z, w) -> rotation matrix
    x, y, z, w = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# ---- NumPy restatement of the front end: visual rates at the IMU times -------------------------------------------------------------
def _nearest(ts, t):                                    # FindClosestTimestamp on sorted times (first strict minimum)
    hi = np.searchsorted(ts, t, side="left"); n = ts.size
    lo, hc = np.clip(hi - 1, 0, n - 1), np.clip(hi, 0, n - 1)
    k = np.where(hi == 0, 0, np.where(hi == n, n - 1, np.where(np.abs(t - ts[lo]) <= np.abs(t - ts[hc]), lo, hc)))
    return k, np.abs(t - ts[k])


def _slerp(a, b, t):                                    # Eigen::Quaternion::slerp
    d = (a * b).sum(-1); ad = np.abs(d); lin = ad >= 1.0 - 2.220446049250313e-16
    th = np.arccos(np.minimum(ad, 1.0)); sth = np.where(lin, 1.0, np.sin(th))
    s0 = np.where(lin, 1.0 - t, np.sin((1.0 - t) * th) / sth)
    s1 = np.where(lin, t, np.sin(t * th) / sth)
    return s0[:, None] * a + np.where(d < 0, -s1, s1)[:, None] * b


def _interp(t_old, q_old, t_new):                       # InterpolateQuaternions: nearest sample, slerp "forwards" by dist / step
    k, dist = _nearest(t_old, t_new)
    k1 = np.minimum(k + 1, t_old.size - 1)
    f = dist / np.where(k1 > k, t_old[k1] - t_old[k], 1.0)
    return np.where((k < t_old.size - 1)[:, None], _slerp(q_old[k], q_old[k1], f), q_old[k])


def _front_end(tv, q_cw, ti, gyro, bias=None):
    """-> dict(t, raw, bad, vis, imu): IMU times in the common window, raw visual rates, their outlier flags, and the 15-tap averages of
    the held visual rates and of the gyroscope."""
    vt, vi = np.unique(tv[::-1], return_index=True); vi = tv.size - 1 - vi           # time order, a repeated time keeps the last
    gt, gi = np.unique(ti[::-1], return_index=True); gi = ti.size - 1 - gi
    imu_dt = np.sum(np.diff(ti)) / (ti.size - 1)                                      # file order
    d = np.sort(np.diff(vt)); cam_dt = (d[d.size // 2 - 1] + d[d.size // 2]) / 2 if d.size % 2 == 0 else d[d.size // 2]
    grid = [vt[0]]
    while grid[-1] + cam_dt < vt[-1]:
        grid.append(grid[-1] + cam_dt)
    grid = np.array(grid); qg = _interp(vt, q_cw[vi], grid)
    g = gyro[gi] - (0.0 if bias is None else np.asarray(bias))
    t0, tend = max(grid[0], gt[0]), max(grid[-1], gt[-1])
    m, mg = (gt >= t0) & (gt <= tend), (grid >= t0) & (grid <= tend)
    t = gt[m] - t0
    qi = _interp(grid[mg] - t0, qg[mg], t)
    dq = np.diff(qi, axis=0); dq = np.vstack([dq, dq[-1:]])
    inv = qi * np.array([-1.0, -1.0, -1.0, 1.0]) / (qi * qi).sum(1)[:, None]
    raw = -2.0 / imu_dt * (dq[:, 3:] * inv[:, :3] + inv[:, 3:] * dq[:, :3] + np.cross(dq[:, :3], inv[:, :3]))
    bad = (np.abs(raw) > 2 * np.pi).any(1)
    held = raw.copy()
    for i in np.flatnonzero(bad):                       # repeat the (repaired) predecessor, zero for i <= 1
        held[i] = held[i - 1] if i > 1 else 0.0

    def sma(x):
        c = np.vstack([np.zeros((1, 3)), np.cumsum(x, 0)]); i = np.arange(x.shape[0]); k0 = np.maximum(i - 14, 0)
        return (c[i + 1] - c[k0]) / (i - k0 + 1)[:, None]
    return dict(t=t, raw=raw, bad=bad, vis=sma(held), imu=sma(g[m]))


def _squared_errors(fe, r):
    """|vis(t_i - offset) - (R imu_i + bias)|^2 at the returned rotation, bias and offset (InterpolateVector3d at the shifted times)."""
    t, vis = fe["t"], fe["vis"]
    k, dist = _nearest(t - r["time_offset_s"], t)
    k1 = np.minimum(k + 1, t.size - 1)
    f = np.where(k1 > k, dist / np.where(k1 > k, t[k1] - t[k], 1.0), 0.0)[:, None]
    v = (1 - f) * vis[k] + f * vis[k1]
    D = v - (fe["imu"] @ _qmat(r["q_gyro_to_cam"]).T + r["gyro_bias"])
    return (D * D).sum(1)


def _runs(bad):
    e = np.flatnonzero(np.diff(np.r_[0, bad.astype(int), 0]))
    return e[1::2] - e[::2]


# ---- the cases ------------------------------------------------------------------------------------------------------------------
def _spin_burst(t1, dur=0.3, amp=1.2):
    """About the camera's z axis, a rotation-vector bump of amp rad over dur s: peak rate amp pi / dur = 12.6 rad/s."""
    def f(t):
        u = np.clip((t - t1) / dur, 0.0, 1.0); a = np.zeros((t.size, 3)); da = np.zeros((t.size, 3))
        a[:, 2] = amp * (1 - np.cos(2 * np.pi * u)) / 2
        da[:, 2] = np.where((u > 0) & (u < 1), amp * np.pi / dur * np.sin(2 * np.pi * u), 0.0)
        return a, da
    return f


def _flipped(tv, q_cw):
    s = np.random.default_rng(11).choice([-1.0, 1.0], tv.size); s[0], s[1] = 1.0, -1.0
    return q_cw * s[:, None]


def _spiked(w):
    """20 bursts of 8 samples (2 % of the stream) with 5 rad/s added in random directions."""
    rng = np.random.default_rng(21); w = w.copy()
    for st in rng.choice(w.shape[0] - 10, 20, replace=False):
        d = rng.normal(size=3); w[st:st + 8] += 5.0 * d / np.linalg.norm(d)
    return w


def _case(name):
    """-> (args, kwargs, truth): truth = (q_ic, offset, which of "q", "td", "bias" the oracle must recover) or None."""
    full = ("q", "td", "bias")
    if name.startswith("mount_"):
        _, m, b = name.split("_")
        args = _analytic(seed=3, fps=60.0, td=TD, q_ic=MOUNTINGS[m])
        return args, (dict(gyro_bias=BIAS) if b == "known" else {}), (MOUNTINGS[m], TD, full)
    base = _analytic(seed=3, fps=60.0, td=TD)
    tv, q_cw, ti, w = base
    rng = np.random.default_rng(2)
    if name == "base":
        return base, {}, (Q_IC, TD, full)
    if name == "burst":                                  # offset 37 ms: the shifted lookup reads the first visual samples
        return _analytic(seed=3, fps=60.0, td=0.037, extra=_spin_burst(0.0)), {}, None
    if name == "flips":
        tvb, qb, tib, wb = _analytic(seed=3, fps=60.0, td=0.037, extra=_spin_burst(0.0))
        return (tvb, _flipped(tvb, qb), tib, wb), {}, None
    if name == "spikes":
        return (tv, q_cw, ti, _spiked(w)), {}, None
    if name == "permuted":                               # first and last gyroscope sample stay put: same file-order period
        pv = rng.permutation(tv.size); pg = np.r_[0, 1 + rng.permutation(ti.size - 2), ti.size - 1]
        return (tv[pv], q_cw[pv], ti[pg], w[pg]), {}, (Q_IC, TD, full)
    if name == "reversed":
        return (tv[::-1], q_cw[::-1], ti[::-1], w[::-1]), {}, None
    if name == "duplicates":                             # earlier copies carry other values; the file-order period shrinks by 0.5 %
        dg, dv = rng.choice(ti.size, 40, replace=False), rng.choice(tv.size, 12, replace=False)
        qg = rng.normal(size=(12, 4)); qg /= np.linalg.norm(qg, axis=1)[:, None]
        return (np.r_[tv[dv], tv], np.r_[qg, q_cw], np.r_[ti[dg], ti], np.r_[w[dg] + rng.normal(size=(40, 3)), w]), {}, (Q_IC, TD, ("q", "td"))
    if name == "irregular":                              # jittered 200 Hz clock, a 0.25 s gap, from 0.5 s before to 0.5 s after the video
        tt = np.arange(-0.5, 40.5, 0.005); tt = tt + 0.0008 * np.sin(1.618 * np.arange(tt.size)); tt = tt[(tt < 17.0) | (tt > 17.25)]
        return _analytic(seed=3, fps=60.0, td=TD, imu_t=tt), {}, None
    if name == "n257":
        return _analytic(seed=3, fps=60.0, td=TD, duration=1.485), {}, None
    if name == "n12":                                    # shorter than the 15-tap moving average
        return _analytic(seed=3, fps=60.0, td=TD, duration=0.26), {}, None
    if name == "imu1khz":                                # 4 minutes: 7200 views, 240 k gyroscope samples
        return _analytic(seed=3, fps=30.0, imu_hz=1000.0, td=TD, duration=240.0), {}, None
    raise KeyError(name)


MOUNT_CASES = [f"mount_{m}_{b}" for m in MOUNTINGS for b in ("estimated", "known")]
OTHER_CASES = ["burst", "flips", "spikes", "permuted", "reversed", "duplicates", "irregular", "n257", "n12", "imu1khz"]


def _check_truth(r, truth, known):
    q_ic, td, what = truth
    if "q" in what:
        assert _qdiff(r["q_gyro_to_cam"], q_ic * CONJ) < 2e-3, r["q_gyro_to_cam"]
    if "td" in what:
        assert abs(r["time_offset_s"] - td) < 0.015, r["time_offset_s"]
    if known:
        assert np.array_equal(r["gyro_bias"], BIAS)
    elif "bias" in what:
        assert np.abs(r["gyro_bias"] + _rot(q_ic * CONJ, BIAS)).max() < 5e-3, r["gyro_bias"]


def _check_parity(rg, ro):
    assert rg["iterations"] == ro["iterations"]
    assert abs(rg["time_offset_s"] - ro["time_offset_s"]) < 1e-12, (rg["time_offset_s"], ro["time_offset_s"])
    assert _qdiff(rg["q_gyro_to_cam"], ro["q_gyro_to_cam"]) < 1e-9, (rg["q_gyro_to_cam"], ro["q_gyro_to_cam"])
    assert np.abs(rg["gyro_bias"] - ro["gyro_bias"]).max() < 1e-9, (rg["gyro_bias"], ro["gyro_bias"])
    assert abs(rg["error"] - ro["error"]) < 1e-9 * ro["error"], (rg["error"], ro["error"])


# ---- CPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MOUNT_CASES + [c for c in OTHER_CASES if c != "imu1khz"])
def test_oracle_on_the_edge_streams(oracle_factory, name):
    args, kw, truth = _case(name)
    r = oracle_factory().estimate_imu_to_camera_rotation(*args, **kw)
    assert r["iterations"] == 18 and np.all(np.isfinite(r["q_gyro_to_cam"])) and abs(np.linalg.norm(r["q_gyro_to_cam"]) - 1) < 1e-12
    if truth is not None:
        _check_truth(r, truth, "gyro_bias" in kw)


def _branch(R):                                         # which case of the trace / largest-diagonal rule R takes
    if np.trace(R) > 0:
        return "trace"
    return "x" if R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2] else ("y" if R[1, 1] > R[2, 2] else "z")


@pytest.mark.parametrize("mount,branch", [("x180", "x"), ("y180", "y"), ("z180", "z"), ("identity", "trace"), ("random", "y")])
def test_mountings_reach_every_branch_of_the_quaternion_rule(oracle_factory, mount, branch):
    """The estimated R_ci of a 180 degree mounting has trace ~ -1 and its largest diagonal on the rotation axis: one mounting per
    trace <= 0 branch of the matrix-to-quaternion rule; identity takes the trace > 0 branch, the random mounting (2.4 rad) the y one."""
    args, kw, _ = _case(f"mount_{mount}_estimated")
    R = _qmat(oracle_factory().estimate_imu_to_camera_rotation(*args, **kw)["q_gyro_to_cam"])
    assert _branch(R) == branch
    if mount.endswith("180"):
        assert np.trace(R) < -0.99


def test_front_end_restatement_matches_the_oracle_on_the_plain_scene(oracle_factory):
    """The NumPy front end is what the two checks below rely on: its squared errors at the oracle's answer give the oracle's robust error
    to the accuracy of the returned offset (the midpoint of the last bracket, not the candidate the error was taken at)."""
    args, _, _ = _case("base")
    r = oracle_factory().estimate_imu_to_camera_rotation(*args)
    e = _squared_errors(_front_end(*args), r)
    assert e.max() < 1.345 and abs(e.sum() - r["error"]) < 0.01 * r["error"]


def test_flips_and_burst_reach_the_hold_rule():
    fe = _front_end(*_case("flips")[0])
    assert not fe["bad"][0] and fe["bad"][1] and fe["bad"][2]          # the "zero for i <= 1" rule, next to an unflagged sample 0
    assert _runs(fe["bad"]).max() >= 3 and fe["bad"].sum() >= 20       # held runs longer than one sample
    assert np.abs(fe["raw"][fe["bad"]]).max() > 10.0
    # the flips themselves negate single finite differences: the raw rates differ from the unflipped burst's at many samples
    fb = _front_end(*_case("burst")[0])
    assert np.sum(np.abs(fe["raw"] - fb["raw"]).max(1) > 0.1) > 100


def test_spikes_reach_the_huber_branch(oracle_factory):
    args, _, _ = _case("spikes")
    e = _squared_errors(_front_end(*args), oracle_factory().estimate_imu_to_camera_rotation(*args))
    assert np.sum(e > 1.345) >= 20


def test_size_cases_have_the_intended_windows():
    assert _front_end(*_case("n257")[0])["t"].size == 257
    assert _front_end(*_case("n12")[0])["t"].size == 12
    tv, _, ti, _ = _case("imu1khz")[0]
    assert tv.size == 7200 and ti.size == 240000 and ti.size > GRID_CAP


def test_twelve_sample_window_ends_on_a_clamped_lookup(oracle_factory):
    """Why the 12-sample case asserts no rotation: at the offset the search ends on, every shifted lookup reads the last visual sample."""
    args, _, _ = _case("n12")
    r = oracle_factory().estimate_imu_to_camera_rotation(*args)
    fe = _front_end(*args)
    k, _ = _nearest(fe["t"] - r["time_offset_s"], fe["t"])
    assert np.all(k == fe["t"].size - 1)


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", MOUNT_CASES + OTHER_CASES)
def test_gpu_matches_oracle_on_the_edge_streams(oracle_factory, gpu_factory, name):
    args, kw, truth = _case(name)
    ro = oracle_factory().estimate_imu_to_camera_rotation(*args, **kw)
    rg = gpu_factory().estimate_imu_to_camera_rotation(*args, **kw)
    if name == "n12":
        # the search ends where the shifted lookups clamp to the last visual samples: the cross-covariance is (nearly) zero, so the
        # optimal rotation is not unique (SVD and Horn's method pick different ones) and the bias and the robust error follow that
        # pick; the bracket decisions, i.e. offset and iteration count, are still the same
        assert rg["iterations"] == ro["iterations"] and abs(rg["time_offset_s"] - ro["time_offset_s"]) < 1e-12
        return
    _check_parity(rg, ro)
    if truth is not None:
        _check_truth(rg, truth, "gyro_bias" in kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name,reference", [("flips", "burst"), ("spikes", "base")])
def test_gpu_held_and_spiked_samples_reach_the_sums(gpu_factory, name, reference):
    """The flipped / spiked stream gives another answer than the same scene without the defect."""
    a = gpu_factory().estimate_imu_to_camera_rotation(*_case(name)[0])
    b = gpu_factory().estimate_imu_to_camera_rotation(*_case(reference)[0])
    assert _qdiff(a["q_gyro_to_cam"], b["q_gyro_to_cam"]) > 1e-4 and abs(a["error"] - b["error"]) > 1e-3 * b["error"]
