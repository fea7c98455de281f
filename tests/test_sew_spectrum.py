"""Spline error weighting (row f2) beyond the three recorded streams of test_sew.py: every bin of the spectrum, the residual energy the
knot-spacing search is built on, and end-to-end runs of the reference's python/sew.py, at lengths where the CUDA path changes shape.

The CUDA spectrum is Bluestein's chirp-z transform on power-of-two Stockham passes of length M = 2^ceil(log2(2N - 1)), so N = 2^k and
2^k + 1 are where M doubles; N = 4 is the smallest M (8); 524289 needs M = 2^21 (268 MB of scratch).  The residual-energy reduction
caps its grid at 4 x 132 SMs x 256 threads = 135168 threads on an H100, so longer streams run its grid-stride loop more than once.

References: a NumPy statement of make_reference_spectrum (np.fft, itself checked against a direct long-double DFT for N <= 4096) and
of the residual energy sum((1 - H(f; dt)) Xhat)^2 with math.fsum.  Inputs are the closed-form streams of tests/sew_signals.py.

Spectrum bar: max_k |dXhat_k| <= 1e-12 ||x||_2 and <= 1e-12 max Xhat over the whole spectrum.  A per-bin relative bar would be wrong:
the gravity-dominated stream has tiny bins next to 9.81 m/s2 of DC.  A NumPy restatement of the same Bluestein (np.fft as the inner
transform) on these streams reaches |dXhat| / ||x|| = 1.9e-13 (tones, N = 524289) and |dXhat| / max Xhat = 2.4e-13 (gravity, N = 7).
Measured on an H100 80GB HBM3 (700 W power limit) against np.fft, over all 66 length / stream pairs: up to 1.2e-13 of ||x|| (jitter,
N = 524289; tones 9.7e-14, gravity 2.5e-14) and up to 1.5e-13 of max Xhat (gravity, N = 257; tones and jitter below 7e-16), i.e. at
the level of the CPU restatement.

Residual energy without an API change: with min_dt = max_dt = d the search returns d, and var * N^2 is sum((1 - H) Xhat)^2 at d,
so the quality (E / N)(1 - q) / (var N) follows too."""
import math
import os

import numpy as np
import pytest

import sew_signals as S

HERE = os.path.dirname(os.path.abspath(__file__))
LENGTHS = (4, 5, 7, 8, 16, 17, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 4097, 65536, 65537, 135168, 135169, 200003, 524289)
GRID_CAP = 4 * 132 * 256                    # threads of one grid-stride pass of the f2 reductions on an H100
assert 135168 == GRID_CAP
FIXTURES = sorted(os.path.join(HERE, "golden", f) for f in os.listdir(os.path.join(HERE, "golden")) if f.startswith("closed_form_sew_"))
RECORDED = sorted(os.path.join(HERE, "golden", f) for f in os.listdir(os.path.join(HERE, "golden")) if f.startswith("sew_") and f.endswith(".npz"))
SETTINGS = (("r3", 0.96, 0.01, 0.15), ("so3", 0.98, 0.01, 0.2))                  # python/get_sew_for_dataset.py:38-48
RESIDUAL_DTS = (0.0025, 0.01, 0.05, 0.2, 3.0)


def _fft_length(n):
    m = 1
    while m < 2 * n - 1:
        m <<= 1
    return m


def _dft_longdouble(x):
    """Xhat of make_reference_spectrum by the direct DFT in long double, twiddles indexed exactly by (k n) mod N."""
    n = x.shape[0]
    ang = np.arange(n, dtype=np.longdouble) * (-2 * np.pi / np.longdouble(n))
    c, s = np.cos(ang), np.sin(ang)
    idx = np.outer(np.arange(n, dtype=np.int64), np.arange(n, dtype=np.int64)) % n
    xl = x.astype(np.longdouble)
    re, im = c[idx] @ xl, s[idx] @ xl                  # (n, 3)
    p = (re * re + im * im).sum(axis=1)
    p[0] = 0
    return np.sqrt(p / 3)


def _freqs(t):
    n = t.size
    return np.fft.fftfreq(n, d=1 / (1 / np.mean(np.diff(t))))


def _residual_energy(Xhat, freqs, dt):
    """sum_k ((1 - H(f_k; dt)) Xhat_k)^2 summed exactly (math.fsum)."""
    v = (1.0 - S.spline_response(freqs, dt)) * Xhat
    return math.fsum(v * v)


def _spectrum_error(spec, ref, x):
    d = float(np.abs(spec - ref).max())
    return d / float(np.linalg.norm(x)), d / float(ref.max())


def test_lengths_cover_the_transform_and_grid_shapes():
    ms = {n: _fft_length(n) for n in LENGTHS}
    assert ms[4] == 8 and ms[524289] == 2 ** 21 and ms[200003] == 2 ** 19
    assert all(ms[2 ** k + 1] == 2 * ms[2 ** k] for k in (2, 4, 5, 8, 10, 16))           # M doubles from 2^k to 2^k + 1
    assert max(LENGTHS) > GRID_CAP and GRID_CAP in LENGTHS and GRID_CAP + 1 in LENGTHS


@pytest.mark.parametrize("kind", S.KINDS)
def test_streams_are_what_they_claim(kind):
    n = 3001
    t, x = S.make(kind, n)
    assert t.shape == (n,) and x.shape == (n, 3) and np.all(np.diff(t) > 0)
    X = S.reference_spectrum(x)
    if kind == "tones":                     # bin-exact tone at k = n // 3 (and its mirror), alternating sequence at the top bin
        k3 = n // 3
        assert X[k3] > 50 * np.median(X) and abs(X[k3] - X[n - k3]) < 1e-9 * X[k3]
        assert X[(n + 1) // 2] > 50 * np.median(X)
    elif kind == "gravity":                 # 9.81 of DC against milli-g vibration
        assert abs(x[:, 2].mean() - 9.81) < 1e-3 and np.abs(x[:, :2] - x[:, :2].mean(0)).max() < 0.03
    else:                                   # one dropped sample on a jittered clock
        d = np.diff(t) * S.RATE
        assert np.sum(d > 1.5) == 1 and 0.9 < d[d < 1.5].min() and d.max() < 2.1 and np.std(d[d < 1.5]) > 1e-3


@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("n", [n for n in LENGTHS if n <= 4096])
def test_numpy_fft_matches_long_double_dft(kind, n):
    t, x = S.make(kind, n)
    ref = _dft_longdouble(x)
    X = S.reference_spectrum(x)
    assert float(np.abs(X - ref).max()) <= 1e-14 * float(np.linalg.norm(x))


@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("n", [n for n in LENGTHS if n <= 4097])
def test_oracle_spectrum_every_bin(oracle_factory, kind, n):
    t, x = S.make(kind, n)
    _, _, spec = oracle_factory().spline_error_weighting(t, x, 0.98, 0.05, 0.05, want_spectrum=True)
    ref = S.reference_spectrum(x)
    e_norm, e_max = _spectrum_error(spec, ref, x)
    assert e_norm <= 1e-12 and e_max <= 1e-12, (e_norm, e_max)


@pytest.mark.parametrize("path", RECORDED, ids=[os.path.basename(p)[:-4] for p in RECORDED])
def test_restated_quality_reproduces_the_recorded_quality(path):
    """The NumPy residual energy here against the reference's own quality function at five spacings (test_sew.py's recordings)."""
    g = np.load(path)
    for tag, key in (("r3", "accel"), ("so3", "gyro")):
        X = S.reference_spectrum(g[key])
        q = float(g[f"q_{tag}"])
        qual = [math.fsum(X * X) * (1 - q) / _residual_energy(X, _freqs(g["times"]), d) for d in g[f"{tag}_quality_dts"]]
        assert np.abs(np.array(qual) - g[f"{tag}_quality"]).max() <= 1e-10 * np.abs(g[f"{tag}_quality"]).max()


def _check_fixed_spacing(api, t, x, q, dts, bar):
    """min_dt = max_dt = d: the search must return d, and var * N^2 must be the residual energy at d of the returned spectrum."""
    n = t.size
    out = []
    for d in dts:
        dt, var, spec = api.spline_error_weighting(t, x, q, d, d, want_spectrum=True)
        assert dt == d
        e_res = _residual_energy(spec, _freqs(t), d)
        assert abs(var * n * n - e_res) <= bar * e_res, (n, d, var * n * n, e_res)
        out.append(math.fsum(spec * spec) / n * (1 - q) / (var * n))
    return np.array(out)


@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("n", (4, 257, 4097))
def test_oracle_residual_energy_at_fixed_spacings(oracle_factory, kind, n):
    t, x = S.make(kind, n)
    _check_fixed_spacing(oracle_factory(), t, x, 0.98, RESIDUAL_DTS, 1e-12)


@pytest.mark.parametrize("path", RECORDED, ids=[os.path.basename(p)[:-4] for p in RECORDED])
def test_oracle_quality_from_fixed_spacing_runs(oracle_factory, path):
    g = np.load(path)
    for tag, key in (("r3", "accel"), ("so3", "gyro")):
        qual = _check_fixed_spacing(oracle_factory(), g["times"], g[key], float(g[f"q_{tag}"]), g[f"{tag}_quality_dts"], 1e-12)
        assert np.abs(qual - g[f"{tag}_quality"]).max() <= 1e-10 * np.abs(g[f"{tag}_quality"]).max()


def test_closed_form_fixtures_span_the_lengths():
    ns = sorted(int(np.load(p)["n"]) for p in FIXTURES)
    assert len(FIXTURES) == 4 and ns[0] <= 20000 and ns[-1] == 524289 and sum(n > GRID_CAP for n in ns) >= 2


def _check_fixture(api, path, check_spectrum=True):
    g = np.load(path)
    t, x = S.make(str(g["kind"]), int(g["n"]))
    for tag, q, lo, hi in SETTINGS:
        dt, var = api.spline_error_weighting(t, x, q, lo, hi)
        ref_dt, ref_var = float(g[f"{tag}_dt"]), float(g[f"{tag}_var"])
        assert abs(dt - ref_dt) <= 1e-9 * ref_dt and abs(var - ref_var) <= 1e-9 * ref_var, (tag, dt, ref_dt, var, ref_var)
        qual = _check_fixed_spacing(api, t, x, q, g["quality_dts"], 1e-12)
        assert np.abs(qual - g[f"{tag}_quality"]).max() <= 1e-9 * np.abs(g[f"{tag}_quality"]).max(), (tag, qual, g[f"{tag}_quality"])
    if check_spectrum:
        _, _, spec = api.spline_error_weighting(t, x, 0.98, 0.05, 0.05, want_spectrum=True)
        assert np.abs(spec[g["bins"]] - g["spectrum"]).max() <= 1e-9 * np.abs(g["spectrum"]).max()


@pytest.mark.parametrize("path", [p for p in FIXTURES if int(np.load(p)["n"]) <= 20000], ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_reproduces_closed_form_fixtures(oracle_factory, path):
    _check_fixture(oracle_factory(), path)


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("n", LENGTHS)
def test_gpu_spectrum_every_bin(gpu_factory, kind, n):
    t, x = S.make(kind, n)
    _, _, spec = gpu_factory().spline_error_weighting(t, x, 0.98, 0.05, 0.05, want_spectrum=True)
    ref = S.reference_spectrum(x)
    e_norm, e_max = _spectrum_error(spec, ref, x)
    print(f"\n[f2 spectrum] {kind} N={n} M={_fft_length(n)}: max|dXhat| = {e_norm:.2e} ||x|| = {e_max:.2e} max Xhat")
    assert spec[0] == 0.0
    assert e_norm <= 1e-12 and e_max <= 1e-12, (e_norm, e_max)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", S.KINDS)
@pytest.mark.parametrize("n", (4, 257, 4097, 135168, 135169, 200003, 524289))
def test_gpu_residual_energy_at_fixed_spacings(gpu_factory, kind, n):
    t, x = S.make(kind, n)
    _check_fixed_spacing(gpu_factory(), t, x, 0.98, RESIDUAL_DTS, 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("path", RECORDED, ids=[os.path.basename(p)[:-4] for p in RECORDED])
def test_gpu_quality_reproduces_the_recorded_quality(gpu_factory, path):
    g = np.load(path)
    for tag, key in (("r3", "accel"), ("so3", "gyro")):
        qual = _check_fixed_spacing(gpu_factory(), g["times"], g[key], float(g[f"q_{tag}"]), g[f"{tag}_quality_dts"], 1e-12)
        assert np.abs(qual - g[f"{tag}_quality"]).max() <= 1e-10 * np.abs(g[f"{tag}_quality"]).max()


@pytest.mark.gpu
@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_gpu_reproduces_closed_form_fixtures(gpu_factory, path):
    _check_fixture(gpu_factory(), path)


# ---- static IMU biases (python/get_imu_biases.py:36-53), same grid-capped reduction shape -------------------------------------
def _biases_fsum(a, g, gravity_const):
    """get_imu_biases.py with exact sums: gravity (as float32) off the dominant mean axis, then the column means."""
    ma = np.array([math.fsum(a[:, d]) / a.shape[0] for d in range(3)])
    mg = np.array([math.fsum(g[:, d]) / g.shape[0] for d in range(3)])
    ax = int(np.argmax(np.abs(ma)))
    grav = np.zeros(3); grav[ax] = float(np.float32(gravity_const * np.sign(ma[ax])))
    return ma - grav, mg, np.abs(ma).max(), np.abs(mg).max()


@pytest.mark.gpu
@pytest.mark.parametrize("n", (1, 255, 257, GRID_CAP + 1, 300001))
def test_gpu_static_biases_against_exact_sums(gpu_factory, n):
    t, acc = S.gravity(n)
    _, gyr = S.jitter(n)
    gyr = gyr + np.array([0.003, -0.002, 0.0015])
    acc = acc[:, [1, 2, 0]] * np.array([1.0, -1.0, 1.0])            # gravity on -y: the sign and the axis search both matter
    ba, bg = gpu_factory().estimate_imu_biases(acc, gyr, 9.81)
    ra, rg, sa, sg = _biases_fsum(acc, gyr, 9.81)
    assert np.abs(ba - ra).max() <= 1e-13 * sa and np.abs(bg - rg).max() <= 1e-13 * sg, (ba - ra, bg - rg)
