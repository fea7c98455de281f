"""Upstream row f3 (SURVEY.md §8(f)): IMU-to-camera rotation + time-offset initialiser,
ImuToCameraRotationEstimator::EstimateCameraImuRotation (src/core/imu_to_camera_rotation_estimator.cc:116-274) with the preparation of
applications/estimate_imu_to_camera_rotation.cc:96-162.

CPU part: the oracle restatement is pinned by an analytic scene (smooth non-periodic rotation R_wc(t) = exp(a(t)), exact body rates
omega_c = Jr(a) a', gyroscope = R_ic omega_c sampled with a known clock offset and bias): it must return R_ci, the offset and the
bias; on BASELINE config 3 (noisy poses, rolling shutter) it must land near the generator's truth.
GPU part (-m gpu): the CUDA path reproduces the oracle (different closed-form rotation solver, atomics in the sums)."""
import numpy as np
import pytest

from openimucameracalibrator_b200 import synthetic as syn

Q_IC = np.array([0.005, -0.007, -0.708, 0.706]); Q_IC /= np.linalg.norm(Q_IC)      # Readme.md:45, x y z w
CONJ = np.array([-1.0, -1.0, -1.0, 1.0])


def _rot(q, v):
    qv = q[:3]; uv = 2.0 * np.cross(qv, v)
    return v + q[3] * uv + np.cross(qv, uv)


def _analytic(duration=40.0, fps=30.0, imu_hz=200.0, td=0.037, bias=(0.004, -0.002, 0.001), seed=0, q_ic=Q_IC, extra=None, imu_t=None):
    """Views, q_cw, gyroscope times and rates of the analytic scene; q_ic is the mounting (x y z w), extra(t) -> (a, da) adds a
    rotation-vector term (a burst), imu_t replaces the regular gyroscope clock."""
    rng = np.random.default_rng(seed)
    f = np.array([0.13, 0.31, 0.47, 0.71, 0.97]); A = rng.uniform(0.05, 0.12, (3, 5)); ph = rng.uniform(0, 2 * np.pi, (3, 5))
    a0 = lambda t: (A[None] * np.sin(2 * np.pi * f[None, None] * t[:, None, None] + ph[None])).sum(-1)                       # noqa: E731
    da0 = lambda t: (A[None] * 2 * np.pi * f[None, None] * np.cos(2 * np.pi * f[None, None] * t[:, None, None] + ph[None])).sum(-1)  # noqa: E731
    a = a0 if extra is None else (lambda t: a0(t) + extra(t)[0])                                                          # noqa: E731
    da = da0 if extra is None else (lambda t: da0(t) + extra(t)[1])                                                       # noqa: E731
    tv = np.arange(int(duration * fps)) / fps
    q_wc = syn.matrix_to_quat_xyzw(syn.so3_exp(a(tv)))
    ti = np.arange(int(duration * imu_hz)) / imu_hz - 0.2 if imu_t is None else np.asarray(imu_t, dtype=np.float64)
    tq = ti + td                                                     # camera-clock time of IMU sample i: t_cam = t_imu + td
    w_c = np.einsum("nij,nj->ni", syn.so3_right_jacobian(a(tq)), da(tq))      # body rate of the camera frame
    w_i = _rot(np.asarray(q_ic, dtype=np.float64), w_c) + np.asarray(bias)           # omega_c = R_ci omega_i (row-wise)
    return tv, q_wc * CONJ, ti, w_i


def _qdiff(a, b):
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def test_oracle_recovers_rotation_offset_and_bias(oracle_factory):
    """The reference's estimator is approximate by construction (nearest-sample interpolation that always steps FORWARD from the
    nearest sample, utils.cc:220-261, makes its objective a sawtooth in the offset with the IMU period): a few milliseconds in
    the offset and a tenth of a degree in the rotation are its accuracy on noise-free data at GoPro-like rates."""
    tv, q_cw, ti, w_i = _analytic(fps=60.0, td=0.1)
    r = oracle_factory().estimate_imu_to_camera_rotation(tv, q_cw, ti, w_i)
    assert r["iterations"] == 18                                       # bracket 2 s -> 1e-4 s at the golden ratio
    assert _qdiff(r["q_gyro_to_cam"], Q_IC * CONJ) < 2e-3              # R_ci: the rotation taking gyroscope to camera rates
    assert abs(r["time_offset_s"] - 0.1) < 0.015
    assert np.abs(r["gyro_bias"] + _rot(Q_IC * CONJ, np.array([0.004, -0.002, 0.001]))).max() < 5e-3    # angVis = R angImu + bias
    # a known bias is subtracted up front and handed back unchanged
    r2 = oracle_factory().estimate_imu_to_camera_rotation(tv, q_cw, ti, w_i, gyro_bias=(0.004, -0.002, 0.001))
    assert np.allclose(r2["gyro_bias"], (0.004, -0.002, 0.001)) and _qdiff(r2["q_gyro_to_cam"], Q_IC * CONJ) < 2e-3
    # a larger clock offset is followed (t_cam = t_imu + offset)
    tv3, q3, ti3, w3 = _analytic(fps=60.0, td=0.3)
    r3 = oracle_factory().estimate_imu_to_camera_rotation(tv3, q3, ti3, w3)
    assert abs((r3["time_offset_s"] - r["time_offset_s"]) - 0.2) < 0.01 and _qdiff(r3["q_gyro_to_cam"], Q_IC * CONJ) < 2e-3
    # input order is irrelevant (std::map semantics)
    p = np.random.default_rng(1).permutation(tv.size)
    r4 = oracle_factory().estimate_imu_to_camera_rotation(tv[p], q_cw[p], ti, w_i)
    assert abs(r4["time_offset_s"] - r["time_offset_s"]) < 1e-12 and _qdiff(r4["q_gyro_to_cam"], r["q_gyro_to_cam"]) < 1e-12


def test_oracle_on_config3_lands_near_the_truth(oracle_factory):
    ds = syn.make_dataset(syn.CONFIGS[3])
    r = oracle_factory().estimate_imu_to_camera_rotation(ds["frame_t"], ds["q_wc"] * CONJ, ds["imu_t"], ds["gyro"])
    q_ci = ds["truth"]["T_i_c"][:4] * CONJ
    assert _qdiff(r["q_gyro_to_cam"], q_ci) < 1e-2
    assert abs(r["time_offset_s"] - ds["time_offset_imu_to_cam_s"]) < 0.03      # mid-exposure of the rolling shutter: ~ half a frame


def test_oracle_rejects_disjoint_streams(oracle_factory):
    tv, q_cw, ti, w_i = _analytic(duration=5.0)
    with pytest.raises(Exception):
        oracle_factory().estimate_imu_to_camera_rotation(tv[:1], q_cw[:1], ti, w_i)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["analytic", "analytic_known_bias", "config3"])
def test_gpu_matches_oracle(oracle_factory, gpu_factory, case):
    if case == "config3":
        ds = syn.make_dataset(syn.CONFIGS[3])
        args = (ds["frame_t"], ds["q_wc"] * CONJ, ds["imu_t"], ds["gyro"]); kw = {}
    else:
        args = _analytic(seed=3, fps=60.0, td=0.1); kw = dict(gyro_bias=(0.004, -0.002, 0.001)) if case.endswith("bias") else {}
    ro = oracle_factory().estimate_imu_to_camera_rotation(*args, **kw)
    rg = gpu_factory().estimate_imu_to_camera_rotation(*args, **kw)
    assert rg["iterations"] == ro["iterations"]
    # identical bracket decisions -> identical offset; a decision can only flip when the two candidate errors tie to ~1e-13
    assert abs(rg["time_offset_s"] - ro["time_offset_s"]) < 1e-12
    assert _qdiff(rg["q_gyro_to_cam"], ro["q_gyro_to_cam"]) < 1e-9 and np.abs(rg["gyro_bias"] - ro["gyro_bias"]).max() < 1e-9
    assert abs(rg["error"] - ro["error"]) < 1e-9 * ro["error"]


@pytest.mark.gpu
def test_gpu_rotation_init_full_size(oracle_factory, gpu_factory):
    """BASELINE config 4 (3000 views, 100 k gyroscope samples): same answer as the oracle; wall time of the whole initialiser incl.
    transfers.  (At 1 kHz the 15-tap averages of the reference's algorithm span less than a frame interval, so the answer itself is
    not meaningful there -- the reference targets 200-400 Hz gyroscopes -- which is why only parity is asserted.)"""
    import time
    ds = syn.make_dataset(syn.CONFIGS[4])
    g = gpu_factory()
    args = (ds["frame_t"], ds["q_wc"] * CONJ, ds["imu_t"], ds["gyro"])
    g.estimate_imu_to_camera_rotation(*args)
    t0 = time.perf_counter(); r = g.estimate_imu_to_camera_rotation(*args); dt = time.perf_counter() - t0
    t1 = time.perf_counter(); ro = oracle_factory().estimate_imu_to_camera_rotation(*args); dto = time.perf_counter() - t1
    assert r["iterations"] == ro["iterations"] == 18
    assert abs(r["time_offset_s"] - ro["time_offset_s"]) < 1e-12 and _qdiff(r["q_gyro_to_cam"], ro["q_gyro_to_cam"]) < 1e-9
    print(f"\n[f3] 3000 views, {ds['imu_t'].size} gyro samples, 18 golden-section steps (36 objective evaluations): "
          f"{dt * 1e3:.2f} ms wall on the GPU, {dto * 1e3:.1f} ms for the single-thread CPU restatement")
