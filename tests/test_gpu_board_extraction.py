"""Radon checkerboard extraction on the GPU (icc_extract_radon_board) against OpenCV's findChessboardCornersSB on committed frames,
against the renderer's truth through four camera models, and for bit-identical results however the frames arrive."""
import os

import numpy as np
import pytest

from openimucameracalibrator_b200 import calibrator, camera_models as cm, synthetic as syn
from openimucameracalibrator_b200._capi import CApi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
W, H, SQ = 14, 9, 0.03
SIZE = (480, 360)
CAMERAS = {
    "pinhole": (cm.PINHOLE, (420.0, 1.0, 0.0, 240.0, 180.0, -0.05, 0.01)),
    "fisheye": (cm.FISHEYE, (220.0, 1.0, 0.0, 238.0, 182.0, 0.05, 0.07, -0.11, 0.05)),
    "double_sphere": (cm.DOUBLE_SPHERE, (240.0, 1.0, 0.0, 236.0, 181.0, -0.215, 0.513)),
    "extended_unified": (cm.EXTENDED_UNIFIED, (210.0, 1.0, 0.0, 241.0, 178.0, 0.5115, 1.062)),
}
# (distance in focal-length units, tilt, tilt axis, roll)
POSES = [(0.55, 0.0, 0.0, 0.0), (0.7, 45.0, 30.0, 90.0), (0.75, 55.0, 100.0, 200.0)]


@pytest.fixture(scope="module")
def api():
    return CApi(calibrator.load_library(), "icc_", 0)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "radon_board_opencv.npz"))


def _render(name, pose, **kw):
    model, intr = CAMERAS[name]
    dist, tilt, axis, roll = pose
    R, t = syn.radon_view_pose(W, H, SQ, dist * intr[0] / 420.0, tilt, axis, roll)
    return syn.render_radon_board(model, intr, SIZE, R, t, W, H, SQ, supersample=3, **kw)


@pytest.fixture(scope="module")
def renders():
    return {(name, k): _render(name, p, blur_sigma_px=0.5) for name in CAMERAS for k, p in enumerate(POSES)}


def _err(uv, truth):
    return np.linalg.norm(uv - truth, axis=-1)


def test_golden_decisions_order_and_accuracy(api, golden):
    frames, found_cv, corners_cv, truth = golden["frames"], golden["found"], golden["corners"], golden["truth"]
    uv, found, s = api.extract_radon_board(frames, W, H)
    assert found.tolist() == found_cv.tolist(), (golden["names"], found, found_cv)
    assert s["n_found"] == found_cv.sum() and s["candidate_overflow"] == 0, s
    for k in np.nonzero(found_cv)[0]:
        d_cv = _err(uv[k], corners_cv[k])
        e_gpu, e_cv = _err(uv[k], truth[k]), _err(corners_cv[k], truth[k])
        print(f"{golden['names'][k]}: |gpu - opencv| max {d_cv.max():.3f} px; rms to truth gpu {np.sqrt((e_gpu ** 2).mean()):.4f} "
              f"opencv {np.sqrt((e_cv ** 2).mean()):.4f}; max gpu {e_gpu.max():.4f} opencv {e_cv.max():.4f}")
        assert d_cv.max() < 1.0                                          # same id order as OpenCV: one square is > 15 px here
        assert np.sqrt((e_gpu ** 2).mean()) <= np.sqrt((e_cv ** 2).mean()) + 0.02
    for k in np.nonzero(~found_cv)[0]:
        assert np.isnan(uv[k]).all()


def test_golden_downsample_matches_cv2_resize(api, golden):
    for f in golden["factors"]:
        ref = golden["resize_" + f"{f:g}".replace(".", "p")]
        _, _, s = api.extract_radon_board(golden["frames"][:1], W, H, float(f))
        assert (s["height"], s["width"]) == ref.shape
    # the pixels themselves are checked byte for byte against cv2.resize in the CPU suite (the kernel runs that same header code);
    # here the corners found at f = 2 must be the f = 1 corners in the halved image's pixels
    uv1, f1, _ = api.extract_radon_board(golden["frames"][:1], W, H, 1.0)
    uv2, f2, _ = api.extract_radon_board(golden["frames"][:1], W, H, 2.0)
    assert f1[0] and f2[0]
    assert np.abs((uv1[0] + 0.5) / 2 - 0.5 - uv2[0]).max() < 0.15


def _cases():
    for name in CAMERAS:
        for k in range(len(POSES)):
            marks = ()
            if (name, k) == ("double_sphere", 1):   # measured: not found (DESIGN 3.10)
                marks = pytest.mark.xfail(strict=True, reason="DoubleSphere view at 45 degrees of tilt, rolled by 90 degrees: not found at 480x360")
            yield pytest.param(name, k, marks=marks, id=f"{name}-{k}")


@pytest.mark.parametrize("name,k", list(_cases()))
def test_noiseless_models_and_poses(api, renders, name, k):
    img, truth, valid = renders[(name, k)]
    assert valid.all()
    uv, found, s = api.extract_radon_board(img, W, H)
    assert found[0], s
    e = _err(uv[0], truth)
    print(f"{name} pose {POSES[k]}: rms {np.sqrt((e ** 2).mean()):.4f} px, max {e.max():.4f} px")
    # measured on an H100 (DESIGN 3.10): rms 0.074-0.154 px; max 0.19 px at 0 degrees of tilt, 0.34 px at 45 and 0.70 px at 55, where
    # the squares are 5 px across along the foreshortened axis and the refinement window shrinks to 2 px
    assert np.sqrt((e ** 2).mean()) <= 0.2 and e.max() <= (0.4 if POSES[k][1] < 50 else 0.75)


def test_blur_and_noise(api):
    imgs, truth = [], []
    for k, p in enumerate(POSES):
        img, uv, ok = _render("pinhole", p, blur_sigma_px=0.8, noise_sigma_dn=2.0, seed=k)
        imgs.append(img); truth.append(uv)
    uv, found, _ = api.extract_radon_board(np.stack(imgs), W, H)
    assert found.all()
    e = _err(uv, np.stack(truth))
    print(f"blur 0.8 px, noise 2 DN: rms {np.sqrt((e ** 2).mean()):.4f} px, max {e.max():.4f} px")
    assert np.sqrt((e ** 2).mean()) <= 0.2


def test_not_found_without_markers_board_or_full_view(api):
    no_markers = _render("pinhole", POSES[0], markers=False, blur_sigma_px=0.5)[0]
    model, intr = CAMERAS["pinhole"]
    R, t = syn.radon_view_pose(W, H, SQ, 0.55, 0.0, 0.0, 0.0, offset_m=(3.0, 0.0))
    no_board = syn.render_radon_board(model, intr, SIZE, R, t, W, H, SQ, supersample=2)[0]
    R, t = syn.radon_view_pose(W, H, SQ, 0.55, 0.0, 0.0, 0.0, offset_m=(0.15, 0.0))
    cut, _, valid = syn.render_radon_board(model, intr, SIZE, R, t, W, H, SQ, supersample=2, blur_sigma_px=0.5)
    assert not valid.all()
    uv, found, s = api.extract_radon_board(np.stack([no_markers, no_board, cut]), W, H)
    assert not found.any() and np.isnan(uv).all(), s
    assert s["n_no_markers"] == 1 and s["n_no_grid"] + s["n_wrong_count"] == 2, s


def test_not_found_when_mirrored_or_markers_moved(api, renders):
    # a board seen from the back (or through a flipped camera) has its markers mirrored; a board whose L of markers sits in another
    # cell is not the radon board: neither is found, and nothing is written for them
    imgs = [np.ascontiguousarray(renders[("pinhole", k)][0][:, ::-1]) for k in range(len(POSES))]
    imgs += [np.ascontiguousarray(renders[("pinhole", k)][0][::-1, :]) for k in range(len(POSES))]
    mi, mj = syn.radon_marker_cell(W, H)
    imgs += [_render("pinhole", POSES[0], blur_sigma_px=0.5, marker_cell=cell)[0] for cell in ((mi, mj + 1), (mi - 1, mj), (mi + 2, mj - 2))]
    uv, found, s = api.extract_radon_board(np.stack(imgs), W, H)
    assert not found.any() and np.isnan(uv).all(), s
    assert s["n_no_markers"] == len(imgs), s


def test_bit_identical_however_frames_arrive(api, renders):
    import torch
    imgs = np.stack([renders[(n, k)][0] for n in CAMERAS for k in range(len(POSES))])
    ref, fref, _ = api.extract_radon_board(imgs, W, H)
    assert fref.sum() >= len(imgs) - 1
    dev, fdev, _ = api.extract_radon_board(torch.from_numpy(imgs).cuda(), W, H)
    np.testing.assert_array_equal(dev, ref); np.testing.assert_array_equal(fdev, fref)
    one = np.concatenate([api.extract_radon_board(im, W, H)[0] for im in imgs])
    np.testing.assert_array_equal(one, ref)
    for chunk in ("1", "5"):
        os.environ["ICC_BOARD_CHUNK_FRAMES"] = chunk
        try:
            np.testing.assert_array_equal(api.extract_radon_board(imgs, W, H)[0], ref)
        finally:
            del os.environ["ICC_BOARD_CHUNK_FRAMES"]
    pitched = np.zeros(imgs.shape[:2] + (imgs.shape[2] + 37,), dtype=np.uint8)
    pitched[:, :, :imgs.shape[2]] = imgs
    np.testing.assert_array_equal(api.extract_radon_board(pitched[:, :, :imgs.shape[2]], W, H)[0], ref)
    tp = torch.from_numpy(pitched).cuda()[:, :, :imgs.shape[2]]
    np.testing.assert_array_equal(api.extract_radon_board(tp, W, H)[0], ref)


def test_board_extractor_scene(api, tmp_path, golden):
    from openimucameracalibrator_b200 import io_formats
    ex = calibrator.BoardExtractor(0.03, W, H)
    ts = np.arange(len(golden["frames"])) * 0.0333 + 1.5
    scene = ex.write(str(tmp_path / "corners.uson"), golden["frames"], ts)
    back = io_formats.ubjson_loads(open(tmp_path / "corners.uson", "rb").read())
    assert back == scene
    assert scene["calibration_board_type"] == 1 and len(scene["scene_pts"]) == W * H
    assert scene["scene_pts"][str(W + 2)] == [0.03, 0.06, 0.0]          # id = i W + j -> (i s, j s, 0)
    assert sorted(scene["views"]) == sorted(io_formats.view_key(float(t)) for t, f in zip(ts, golden["found"]) if f)
