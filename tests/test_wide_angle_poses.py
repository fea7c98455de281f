"""Board poses from unit bearings with the local tangent reprojection error (icc_set_pose_error(ICC_POSE_ERROR_TANGENT)), the opt-in
residual of the per-view pose step for wide-angle lenses whose corners lie 90 degrees or more off the optical axis.

CPU part: the product's bearing header compiled for the CPU inverts the NumPy camera models; its tangent error has the stated Jacobians,
reduces to the normalised error at b = e_z and does not depend on the basis; the tangent-mode oracle (tests/wide_angle_support.py)
recovers exact poses of boards 70-105 degrees off-axis, keeps a view the default path loses, is more accurate than the default path on
noisy wide views, and keeps the reference's drop rules; the CLIs parse --pose_error.
GPU part (-m gpu): the CUDA path through the C-ABI reproduces the oracle (validity bit-for-bit, poses to 1e-9 noise-free / 2e-8 noisy),
also at full size (3000 views x 144 corners) and through the pose CLI."""
import json
import os
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import _capi as capi
from openimucameracalibrator_b200 import camera_models as cm
from openimucameracalibrator_b200 import io_formats as iof
from openimucameracalibrator_b200 import synthetic as syn
from test_camera_models import CASES
from test_pose_estimation import W, H, _board, _qdiff, _scene
from wide_angle_support import (PoseOracle, oracle_basis, oracle_bearings, product_bearings, product_tangent_basis, product_tangent_error)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "openimucameracalibrator_b200", "bin")
POSE_CLI = os.path.join(BIN, "estimate_camera_poses_from_checkerboard")
HOT_CLI = os.path.join(BIN, "continuous_time_imu_to_camera_calibration")

# two wide cameras the project supports: rays 99 / 100 degrees off-axis at the corners of the 960 x 540 image
WIDE = [(cm.DOUBLE_SPHERE, np.array([200.0, 1.0, 0.0, 472.6, 273.9, -0.215, 0.513])),
        (cm.EXTENDED_UNIFIED, np.array([250.0, 1.0, 0.0, 489.5, 272.0, 0.5115, 1.062]))]
WIDE_IDS = ["wide_DOUBLE_SPHERE", "wide_EXTENDED_UNIFIED"]
ALL = list(CASES) + WIDE
ALL_IDS = [cm.MODEL_NAMES[m] for m, _ in CASES] + WIDE_IDS


def _rot(R):
    return syn.matrix_to_quat_xyzw(R[None])[0]


def _view(rng, model, k, board, ang, dist=(0.35, 0.5), tilt=0.5):
    """One camera pose looking at a board whose centre is `ang` degrees (range) off the optical axis -> (q_wc, p_wc, uv) or None."""
    th, ph = np.radians(rng.uniform(*ang)), rng.uniform(0, 2 * np.pi)
    u = np.array([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)])
    centre = rng.uniform(*dist) * u
    nz = -u + rng.uniform(-tilt, tilt, 3); nz /= np.linalg.norm(nz)              # board normal roughly towards the camera
    nx = np.cross(nz, rng.normal(size=3)); nx /= np.linalg.norm(nx)
    R_cw = np.stack([nx, np.cross(nz, nx), nz], 1)                              # board (world) axes in the camera frame
    pc = board[:, :3] @ R_cw.T + centre
    px, valid = cm.project(model, k, pc)
    if not valid.all():
        return None
    return _rot(R_cw.T), -R_cw.T @ centre, px


def wide_scene(model, k, n_frames=12, seed=0, noise_px=0.0, ang=(70.0, 105.0), board=None):
    rng = np.random.default_rng(seed)
    board = _board() if board is None else board
    C = board.shape[0]
    q, p, uv = [], [], []
    while len(q) < n_frames:
        v = _view(rng, model, k, board, ang)
        if v is None:
            continue
        q.append(v[0]); p.append(v[1]); uv.append(v[2] + rng.normal(0, noise_px, v[2].shape))
    off = (np.arange(n_frames + 1) * C).astype(np.int32)
    return board, off, np.tile(np.arange(C, dtype=np.int32), n_frames), np.concatenate(uv), np.array(q), np.array(p)


def _tangent(api, model, k, board):
    api.set_camera(model, k, W, H); api.set_board_points(board); api.set_pose_error("tangent")
    return api


def _rot_err(q, q_true):
    """rotation angle between two batches of unit quaternions (rad)"""
    return 2 * np.arccos(np.clip(np.abs(np.sum(q * q_true, 1)), 0, 1))


# ---- 1. bearing un-projection ------------------------------------------------------------------------------------------------------
def _rays(model, k, seed):
    """unit rays over the model's field: 0-50 degrees for every model, 90-110 degrees too for the wide cameras, 0-89 for the fisheye"""
    rng = np.random.default_rng(seed)
    hi = {cm.FISHEYE: 89.0}.get(model, 50.0)
    th = [rng.uniform(0, hi, 300)]
    if any(model == m and np.array_equal(k, kk) for m, kk in WIDE):
        th.append(rng.uniform(90, 110, 300))
    th = np.radians(np.concatenate(th)); ph = rng.uniform(0, 2 * np.pi, th.size)
    return np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1)


@pytest.mark.parametrize("model,k", ALL, ids=ALL_IDS)
def test_bearings_invert_the_numpy_models(model, k):
    rays = _rays(model, k, model + 40)
    px, valid = cm.project(model, k, rays)
    assert valid.all()
    for name, (b, ok) in (("product", product_bearings(model, k, px)), ("oracle", oracle_bearings(model, k, px))):
        assert ok.all(), name
        assert np.abs(np.linalg.norm(b, axis=1) - 1).max() < 1e-14, name
        assert np.abs(b - rays).max() < 1e-10, (name, np.abs(b - rays).max())
    if model in (cm.DOUBLE_SPHERE, cm.EXTENDED_UNIFIED) and rays[:, 2].min() < 0:
        assert (product_bearings(model, k, px)[0][:, 2] < 0).sum() >= 250       # past 90 degrees: z < 0


def test_fisheye_bearings_stay_in_front():
    model, k = next(c for c in CASES if c[0] == cm.FISHEYE)
    rays = _rays(model, k, 3)
    px, _ = cm.project(model, k, rays)
    b, ok = product_bearings(model, k, px)
    assert ok.all() and (b[:, 2] > 0).all()
    bm, okm = product_bearings(model, k, cm.project(model, k, -rays)[0])    # -p projects to the pixel of p: the ray is still p
    assert okm.all() and np.abs(bm - rays).max() < 1e-10


# ---- 2. tangent residual -----------------------------------------------------------------------------------------------------------
def test_tangent_error_jacobians_match_central_differences():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(7)
    for i in range(40):
        b = rng.normal(size=3) if i else np.array([0.0, 0.0, -1.0])
        b /= np.linalg.norm(b)
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        R = Rotation.from_quat(q).as_matrix()
        X = rng.normal(0, 0.1, 3)
        t = 0.5 * b - R @ X + rng.normal(0, 0.05, 3)                            # d = R X + t close to the ray
        r, front, J, P = product_tangent_error(b, q, X, t)
        assert front
        h = 1e-6
        for j in range(6):
            dp = np.zeros(6); dp[j] = h
            def at(s):
                Rq = Rotation.from_matrix(R @ Rotation.from_rotvec(s * dp[:3]).as_matrix()).as_quat()
                return product_tangent_error(b, Rq, X, t + s * dp[3:])[0]
            assert np.abs((at(1) - at(-1)) / (2 * h) - J[:, j]).max() < 1e-6 * max(1.0, np.abs(J).max())
        for j in range(3):
            dX = np.zeros(3); dX[j] = h
            num = (product_tangent_error(b, q, X + dX, t)[0] - product_tangent_error(b, q, X - dX, t)[0]) / (2 * h)
            assert np.abs(num - P[:, j]).max() < 1e-6 * max(1.0, np.abs(P).max())
    # behind the ray: front is false
    assert not product_tangent_error(np.array([0.0, 0.0, 1.0]), np.array([0, 0, 0, 1.0]), np.zeros(3), np.array([0.1, 0.0, -1.0]))[1]


def test_tangent_error_is_the_normalised_error_on_the_axis():
    rng = np.random.default_rng(8)
    e1, e2 = product_tangent_basis(np.array([0.0, 0.0, 1.0]))
    assert np.array_equal(e1, [1, 0, 0]) and np.array_equal(e2, [0, 1, 0])
    for _ in range(20):
        d = np.array([*rng.normal(0, 0.3, 2), rng.uniform(0.2, 2.0)])
        r, front, _, _ = product_tangent_error(np.array([0.0, 0.0, 1.0]), np.array([0, 0, 0, 1.0]), d, np.zeros(3))
        assert front and np.array_equal(r, d[:2] * (1.0 / d[2]))           # bit for bit the normalised error pose_system forms


def test_tangent_error_norm_does_not_depend_on_the_basis():
    rng = np.random.default_rng(9)
    b = rng.normal(size=(200, 3)); b /= np.linalg.norm(b, axis=1, keepdims=True)
    b[0] = [0, 0, -1]; b[1] = [0, 0, 1]; b[2] = [1, 0, 0]; b[3] = [0, 0, -1 + 1e-17]
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    d = b + rng.normal(0, 0.05, b.shape)
    o1, o2 = oracle_basis(b)
    for i in range(b.shape[0]):
        e1, e2 = product_tangent_basis(b[i])
        G = np.stack([e1, e2, b[i]])
        assert np.abs(G @ G.T - np.eye(3)).max() < 1e-14 and np.linalg.det(G) > 0        # orthonormal and well conditioned everywhere
        r = product_tangent_error(b[i], np.array([0, 0, 0, 1.0]), d[i], np.zeros(3))[0]
        ro = np.array([o1[i] @ d[i], o2[i] @ d[i]]) / (b[i] @ d[i])
        assert abs(np.linalg.norm(r) - np.linalg.norm(ro)) < 1e-14
        # a rotated basis (e1 cos a + e2 sin a, ...) gives a rotated r of the same length
        a = rng.uniform(0, 2 * np.pi)
        ra = np.array([(np.cos(a) * e1 + np.sin(a) * e2) @ d[i], (-np.sin(a) * e1 + np.cos(a) * e2) @ d[i]]) / (b[i] @ d[i])
        assert abs(np.linalg.norm(ra) - np.linalg.norm(r)) < 1e-14


# ---- 3.-6. the tangent-mode oracle -------------------------------------------------------------------------------------------------
def _scene_for(model, k, seed, **kw):
    if any(model == m and np.array_equal(k, kk) for m, kk in WIDE):
        return wide_scene(model, k, seed=seed, **kw)
    return _scene(model, k, seed=seed, **kw)


@pytest.mark.parametrize("model,k", ALL, ids=ALL_IDS)
def test_oracle_tangent_recovers_exact_poses(model, k):
    board, off, ids, uv, q_true, p_true = _scene_for(model, k, seed=model + 50)
    q, p, e, v = _tangent(PoseOracle(), model, k, board).estimate_board_poses(off, ids, uv)
    assert v.all()
    assert _qdiff(q, q_true).max() < 1e-9 and np.abs(p - p_true).max() < 1e-9 and e.max() < 1e-10


def _lost_view(model, k, seed=0):
    """a view with fewer than 6 corners within 90 degrees of the axis, every corner a valid projection"""
    rng = np.random.default_rng(seed)
    board = _board()
    while True:
        v = _view(rng, model, k, board, (100.0, 104.0), dist=(0.3, 0.35), tilt=0.2)
        if v is None:
            continue
        b, ok = oracle_bearings(model, k, v[2])
        if ok.all() and (b[:, 2] > 0).sum() < 6:
            return v


@pytest.mark.parametrize("model,k", WIDE, ids=WIDE_IDS)
def test_view_the_default_path_loses_is_kept(oracle_factory, model, k):
    board, off, ids, uv, q_true, p_true = wide_scene(model, k, n_frames=3, seed=11, ang=(60.0, 75.0))
    qv, pv, uvv = _lost_view(model, k, seed=model)
    C = board.shape[0]
    off2 = np.r_[off, off[-1] + C].astype(np.int32); ids2 = np.r_[ids, np.arange(C, dtype=np.int32)]; uv2 = np.r_[uv, uvv]
    o = oracle_factory(); o.set_camera(model, k, W, H); o.set_board_points(board)
    assert o.estimate_board_poses(off2, ids2, uv2)[3][3] == 0
    q, p, e, v = _tangent(PoseOracle(), model, k, board).estimate_board_poses(off2, ids2, uv2)
    assert v.tolist() == [1, 1, 1, 1]
    assert _qdiff(q[3:], qv[None]).max() < 1e-9 and np.abs(p[3] - pv).max() < 1e-9


@pytest.mark.parametrize("model,k", WIDE, ids=WIDE_IDS)
def test_tangent_is_more_accurate_on_noisy_wide_views(oracle_factory, model, k):
    board, off, ids, uv, q_true, p_true = wide_scene(model, k, n_frames=30, seed=model + 60, noise_px=0.3, ang=(55.0, 90.0))
    o = oracle_factory(); o.set_camera(model, k, W, H); o.set_board_points(board)
    qn, pn, en, vn = o.estimate_board_poses(off, ids, uv)
    qt, pt, et, vt = _tangent(PoseOracle(), model, k, board).estimate_board_poses(off, ids, uv)
    both = (vn > 0) & (vt > 0)
    assert vt.sum() >= vn.sum() and both.sum() >= 10
    rn, rt = np.median(_rot_err(qn[both], q_true[both])), np.median(_rot_err(qt[both], q_true[both]))
    dn, dt = np.median(np.linalg.norm(pn[both] - p_true[both], axis=1)), np.median(np.linalg.norm(pt[both] - p_true[both], axis=1))
    assert rt < rn and dt < dn, (rt, rn, dt, dn)


def test_oracle_tangent_drop_rules_and_outliers():
    model, k = CASES[0]
    board, off, ids, uv, q_true, p_true = _scene(model, k, n_frames=4, seed=5)
    C = board.shape[0]
    keep = np.ones(uv.shape[0], bool); keep[C + 7:2 * C] = False
    keep[2 * C:3 * C] = False; keep[2 * C + np.array([0, 4, 8, 13, 22, 31, 44, 62])] = True
    off2 = np.array([0, C, C + 7, C + 15, 2 * C + 15], np.int32)
    uv2, ids2 = uv[keep].copy(), ids[keep]
    uv2[off2[3] + 3] += 50.0; uv2[off2[3] + 40] -= 50.0
    q, p, e, v = _tangent(PoseOracle(), model, k, board).estimate_board_poses(off2, ids2, uv2)
    assert v.tolist() == [1, 0, 1, 1]
    assert np.abs(p[[0, 2, 3]] - p_true[[0, 2, 3]]).max() < 1e-8 and _qdiff(q[[0, 2, 3]], q_true[[0, 2, 3]]).max() < 1e-8
    assert (q[1] == [0, 0, 0, 1]).all() and (p[1] == 0).all()
    # a non-planar target is refused (the start is the planar homography)
    bad = board.copy(); bad[5, 2] = 0.01
    assert not _tangent(PoseOracle(), model, k, bad).estimate_board_poses(off, ids, uv)[3].any()


def test_oracle_tangent_board_point_optimisation():
    model, k = WIDE[0]
    board, off, ids, uv, q_true, p_true = wide_scene(model, k, n_frames=40, seed=3)
    o = _tangent(PoseOracle(), model, k, board)
    q, p, e, v, B, n = o.optimize_board_points(off, ids, uv, q_true, p_true, np.ones(40, np.int32))
    assert n == board.shape[0] and v.all()
    assert np.abs(B[:, :3] - board[:, :3]).max() < 1e-10 and np.abs(p - p_true).max() < 1e-9 and e.max() < 1e-10


# ---- 7. CLI flags ------------------------------------------------------------------------------------------------------------------
def test_pose_error_flag_is_parsed_and_checked(tmp_path):
    for cli in (POSE_CLI, HOT_CLI):
        assert os.path.exists(cli), "build the CLI first (__graft_entry__.build())"
        for bad in ("--pose_error=pinhole", "--pose_error=Tangent", "--pose_error="):
            out = subprocess.run([cli, bad], capture_output=True, text=True)
            assert out.returncode == 1 and "--pose_error must be 'normalized' or 'tangent'" in out.stderr, (cli, bad, out.stderr)
    out = subprocess.run([POSE_CLI, "--pose_error", "tangent", "--input_corners=/nonexistent.uson"], capture_output=True, text=True)
    assert out.returncode == 1 and "Failed to load" in out.stderr
    ds = syn.make_dataset(syn.tiny_config())
    paths = iof.write_dataset_files(ds, str(tmp_path))
    base = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items() if a != "input_pose_dataset"] + ["--parse_only"]
    runs = [subprocess.run(base + extra, capture_output=True, text=True) for extra in ([], ["--pose_error=normalized"], ["--pose_error", "tangent"])]
    assert all(r.returncode == 0 for r in runs), [r.stderr for r in runs]
    assert runs[0].stdout == runs[1].stdout == runs[2].stdout


def test_pose_error_is_checked_by_the_library():
    from openimucameracalibrator_b200 import calibrator
    h = capi.CApi(calibrator.load_library(), "icc_", -1)          # host state: a host-only handle takes it
    h.set_pose_error(capi.POSE_ERROR_TANGENT); h.set_pose_error("normalized")
    for bad in (2, -1):
        with pytest.raises(capi.IccError, match="ICC_ERR_INVALID_ARGUMENT"):
            h.set_pose_error(bad)
    h.set_camera(*WIDE[0], W, H)
    with pytest.raises(capi.IccError, match="ICC_ERR_NO_DEVICE"):
        h.pixels_to_bearings(np.zeros((2, 2)))


# ---- GPU -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("model,k", ALL, ids=ALL_IDS)
def test_gpu_bearings_match_oracle(gpu_factory, model, k):
    rng = np.random.default_rng(model + 70)
    px = np.stack([rng.uniform(0, W, 500), rng.uniform(0, H, 500)], -1)
    g = gpu_factory(); g.set_camera(model, k, W, H)
    bg, okg = g.pixels_to_bearings(px)
    bo, oko = oracle_bearings(model, k, px)
    assert (okg == oko).all() and oko.sum() > 400
    m = oko.astype(bool)
    assert np.abs(bg[m] - bo[m]).max() < 1e-12
    bc, okc = product_bearings(model, k, px)                     # the same header on the CPU
    assert (okc == okg).all() and np.abs(bc[m] - bg[m]).max() < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("model,k", ALL, ids=ALL_IDS)
def test_gpu_tangent_poses_match_oracle(gpu_factory, model, k):
    for noise, tol in ((0.0, 1e-9), (0.2, 2e-8)):
        board, off, ids, uv, q_true, p_true = _scene_for(model, k, seed=model + 80, noise_px=noise, n_frames=40)
        uv[off[7] + 11] += 60.0                                     # one gross outlier in view 7
        qo, po, eo, vo = _tangent(PoseOracle(), model, k, board).estimate_board_poses(off, ids, uv)
        qg, pg, eg, vg = _tangent(gpu_factory(), model, k, board).estimate_board_poses(off, ids, uv)
        assert (vo == vg).all() and vo.all()
        assert _qdiff(qg, qo).max() < tol and np.abs(pg - po).max() < tol and np.abs(eg - eo).max() < 1e-10
        assert _qdiff(qg, q_true).max() < 1.5e-2 and np.abs(pg - p_true).max() < 1.5e-2


@pytest.mark.gpu
def test_gpu_tangent_drop_rules_and_lost_view(oracle_factory, gpu_factory):
    model, k = CASES[0]
    board, off, ids, uv, q_true, p_true = _scene(model, k, n_frames=3, seed=9)
    C = board.shape[0]
    keep = np.ones(uv.shape[0], bool); keep[C + 7:2 * C] = False
    off2 = np.array([0, C, C + 7, 2 * C + 7], np.int32)
    q, p, e, v = _tangent(gpu_factory(), model, k, board).estimate_board_poses(off2, ids[keep], uv[keep])
    assert v.tolist() == [1, 0, 1] and (q[1] == [0, 0, 0, 1]).all()
    assert np.abs(p[[0, 2]] - p_true[[0, 2]]).max() < 1e-8
    model, k = WIDE[0]
    qv, pv, uvv = _lost_view(model, k)
    board = _board(); ids1 = np.arange(C, dtype=np.int32); off1 = np.array([0, C], np.int32)
    g = gpu_factory(); g.set_camera(model, k, W, H); g.set_board_points(board)
    assert g.estimate_board_poses(off1, ids1, uvv)[3][0] == 0                    # the default path loses it
    g.set_pose_error("tangent")
    q, p, e, v = g.estimate_board_poses(off1, ids1, uvv)
    assert v[0] == 1 and _qdiff(q, qv[None]).max() < 1e-9 and np.abs(p[0] - pv).max() < 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("model,k", [CASES[4], WIDE[0]], ids=[cm.MODEL_NAMES[CASES[4][0]], WIDE_IDS[0]])
def test_gpu_tangent_board_point_optimisation_matches_oracle(gpu_factory, model, k):
    board, off, ids, uv, q_true, p_true = _scene_for(model, k, n_frames=60, seed=4, noise_px=0.1)
    uv[off[9] + 20] += 40.0
    bad = board.copy(); bad[:, :3] += np.random.default_rng(1).normal(0, 5e-4, (board.shape[0], 3))
    o, g = _tangent(PoseOracle(), model, k, bad), _tangent(gpu_factory(), model, k, bad)
    qo, po, eo, vo = o.estimate_board_poses(off, ids, uv)
    qg, pg, eg, vg = g.estimate_board_poses(off, ids, uv)
    assert (vo == vg).all() and vo.all()
    ro = o.optimize_board_points(off, ids, uv, qo, po, vo)
    rg = g.optimize_board_points(off, ids, uv, qg, pg, vg)
    assert rg[5] == ro[5] == board.shape[0] and (rg[3] == ro[3]).all() and ro[3].all()
    assert np.abs(rg[4] - ro[4]).max() < 1e-8 and np.abs(rg[1] - ro[1]).max() < 1e-7 and _qdiff(rg[0], ro[0]).max() < 1e-7
    assert np.abs(rg[2] - ro[2]).max() < 1e-9 and rg[2].mean() < 0.5 * eg.mean()
    assert np.array_equal(g.get_board_points(), rg[4])


@pytest.mark.gpu
def test_gpu_tangent_full_size(gpu_factory):
    """3000 views x 144 corners on the wide DoubleSphere camera: every view valid, a 40-view sample equals the oracle."""
    import time
    model, k = WIDE[0]
    board = _board(12, 12, 0.015)
    board, off, ids, uv, q_true, p_true = wide_scene(model, k, n_frames=3000, seed=12, noise_px=0.3, ang=(0.0, 100.0), board=board)
    g = _tangent(gpu_factory(), model, k, board)
    g.estimate_board_poses(off, ids, uv)                                          # warm-up (allocations)
    t0 = time.perf_counter()
    q, p, e, v = g.estimate_board_poses(off, ids, uv)
    dt = time.perf_counter() - t0
    assert v.all() and np.isfinite(q).all()
    assert np.median(np.linalg.norm(p - p_true, axis=1)) < 5e-3
    n = 40
    o = _tangent(PoseOracle(), model, k, board)
    qo, po, eo, vo = o.estimate_board_poses(off[: n + 1], ids[: off[n]], uv[: off[n]])
    assert vo.all() and _qdiff(q[:n], qo).max() < 2e-8 and np.abs(p[:n] - po).max() < 2e-8
    print(f"\n[f1 tangent] 3000 views x 144 corners: {dt * 1e3:.2f} ms wall incl. H2D/D2H")


@pytest.mark.gpu
def test_gpu_pose_cli_tangent_end_to_end(tmp_path, gpu_factory):
    model, k = WIDE[0]
    ds = syn.make_dataset(syn.tiny_config())
    board, off, ids, uv, q_true, p_true = wide_scene(model, k, n_frames=30, seed=21, noise_px=0.2, ang=(40.0, 100.0))
    n = len(off) - 1
    ds = dict(ds, model=model, intrinsics=k, image_size=(W, H), board_xyzw=board, corner_offsets=off, point_ids=ids, uv=uv,
              frame_t=ds["frame_t"][:n], q_wc=q_true, p_wc=p_true)
    paths = iof.write_dataset_files(ds, str(tmp_path))
    outs = {}
    for name, extra in (("none", []), ("normalized", ["--pose_error=normalized"]), ("tangent", ["--pose_error", "tangent"])):
        pj = str(tmp_path / f"poses_{name}.json")
        r = subprocess.run([POSE_CLI, "--input_corners=" + paths["input_corners"], "--camera_calibration_json=" + paths["camera_calibration_json"],
                            "--output_pose_dataset=" + pj] + extra, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr + r.stdout
        outs[name] = (open(pj, "rb").read(), r.stdout)
    assert outs["none"] == outs["normalized"]
    assert "mean tangent reprojection error" in outs["tangent"][1]
    pd = json.loads(outs["tangent"][0]); pn = json.loads(outs["none"][0])
    assert len(pd["views"]) > len(pn["views"])
    # the poses are those of the C-ABI call on the file contents, after the tool's camera-height filter (FilterBadPoses)
    d2 = iof.dataset_from_files(ds)
    g = _tangent(gpu_factory(), d2["model"], d2["intrinsics"], d2["board_xyzw"])
    q, p, e, v = g.estimate_board_poses(d2["corner_offsets"], d2["point_ids"], d2["uv"])
    assert v.all()
    v = g.filter_bad_poses(p, v)
    names = [str(int(t * 1e6)) for t in d2["frame_t"]]
    for i, nm in enumerate(names):
        assert (nm in pd["views"]) == bool(v[i])
        if v[i]:
            assert np.abs(np.array(pd["views"][nm]["p_wc"]) - p[i]).max() < 1e-12
    # the hot CLI accepts the tangent pose dataset
    args = [HOT_CLI] + [f"--{a}={b}" for a, b in paths.items() if a != "input_pose_dataset"] + ["--input_pose_dataset=" + str(tmp_path / "poses_tangent.json"), "--parse_only"]
    r = subprocess.run(args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert json.loads(r.stdout)["views"] == len(pd["views"])
