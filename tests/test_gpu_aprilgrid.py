"""AprilGrid extraction on the GPU (icc_extract_aprilgrid) against OpenCV's ArUco detector and cornerSubPix on committed frames,
against the renderer's truth through four camera models, one case per wrapper rule, bit-identical results however the frames
arrive, and the corner file through calibrate_camera and estimate_camera_poses_from_checkerboard."""
import json
import os
import subprocess

import numpy as np
import pytest

from openimucameracalibrator_b200 import calibrator, camera_models as cm, io_formats, synthetic as syn
from openimucameracalibrator_b200._capi import CApi

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(os.path.dirname(HERE), "openimucameracalibrator_b200", "bin")
NX = NY = 6
S = 0.04
SIZE = (960, 540)
CV_TO_REF = [1, 0, 3, 2]    # corner i of the reference's order is OpenCV's corner CV_TO_REF[i] (DESIGN.md "AprilGrid corners")
CAMERAS = {
    "pinhole": (cm.PINHOLE, (820.0, 1.0, 0.0, 480.0, 270.0, -0.05, 0.01)),
    "fisheye": (cm.FISHEYE, (430.0, 1.0, 0.0, 478.0, 272.0, 0.05, 0.07, -0.11, 0.05)),
    "double_sphere": (cm.DOUBLE_SPHERE, (460.0, 1.0, 0.0, 476.0, 271.0, -0.215, 0.513)),
    "extended_unified": (cm.EXTENDED_UNIFIED, (410.0, 1.0, 0.0, 481.0, 268.0, 0.5115, 1.062)),
}


@pytest.fixture(scope="module")
def api():
    return CApi(calibrator.load_library(), "icc_", 0)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "aprilgrid_opencv.npz"))


def _render(name, dist=0.55, tilt=0.0, axis=0.0, roll=0.0, offset=(0.0, 0.0), supersample=3, **kw):
    model, intr = CAMERAS[name]
    R, t = syn.aprilgrid_view_pose(kw.pop("nx", NX), kw.pop("ny", NY), S, dist * intr[0] / 820.0, tilt, axis, roll, offset)
    return syn.render_aprilgrid(model, intr, SIZE, R, t, kw.pop("tags_x", NX), kw.pop("tags_y", NY), S, supersample=supersample, **kw)


def test_opencv_frames(api, golden):
    frames, truth = golden["frames"], golden["truth"]
    uv, status, found, s = api.extract_aprilgrid(frames, NX, NY)
    print(s)
    assert s["quad_overflow"] == 0
    for f in range(len(frames)):
        sel = golden["cv_frame"] == f
        ids, raw, ref = golden["cv_ids"][sel], golden["cv_corners"][sel], golden["cv_refined"][sel]
        # the border rule on the true corners: ArUco's own corners are 1-2 px off, and a tag within 0.3 px of the 4 px limit may go
        # either way (partial_right's tag 8 has a true corner at y = 536.95 > 540 - 4, where ArUco puts 536.0)
        def margin(k):
            q = truth[f, 4 * ids[k]:4 * ids[k] + 4]
            return min(q[:, 0].min(), q[:, 1].min(), SIZE[0] - q[:, 0].max(), SIZE[1] - q[:, 1].max()) - 4.0
        inside = [k for k in range(len(ids)) if ids[k] < 36 and margin(k) > 0.3]
        expect = len(inside) >= 4 and len(set(ids[inside].tolist())) == len(inside)
        assert found[f] == expect, (golden["names"][f], found[f], len(inside))
        if not expect:
            assert (status[f] == 0).all()
            continue
        seen = status[f] != 0
        ours = sorted(set(np.nonzero(seen)[0] >> 2))
        for k in inside:            # every tag OpenCV decodes inside the border is found with the same id
            assert ids[k] in ours, (golden["names"][f], ids[k])
            for i in range(4):
                pid = (ids[k] << 2) + i
                r = ref[k][CV_TO_REF[i]]
                if status[f, pid] == 1 and np.linalg.norm(r - truth[f, pid]) < 0.25:   # where OpenCV's refinement found the junction
                    assert np.linalg.norm(uv[f, pid] - r) < 0.5, (golden["names"][f], pid, uv[f, pid], r)
        kept = status[f] == 1
        e = np.linalg.norm(uv[f][kept] - truth[f][kept], axis=1)
        print(f"{golden['names'][f]}: {len(ours)} tags ({len(inside)} by OpenCV), {kept.sum()} corners kept, {(status[f] == -1).sum()} moved; "
              f"error to truth rms {np.sqrt((e ** 2).mean()):.4f} max {e.max():.4f} px")
        assert e.max() < 0.5
        assert kept.sum() >= 0.9 * seen.sum()
    assert found.sum() == s["n_found"] and (status == 1).sum() == s["n_corners_kept"]


@pytest.mark.parametrize("name", list(CAMERAS))
def test_noise_free_models(api, name):
    imgs, truths = [], []
    for pose in ((0.55, 0.0, 0.0, 0.0), (0.6, 30.0, 20.0, 60.0), (0.6, 25.0, 110.0, 200.0)):
        img, uv, ok = _render(name, *pose, supersample=4)
        imgs.append(img); truths.append(uv)
    uv, status, found, s = api.extract_aprilgrid(np.stack(imgs), NX, NY)
    assert found.all(), s
    kept = status == 1
    e = np.linalg.norm(uv[kept] - np.stack(truths)[kept], axis=1)
    print(f"{name}: {kept.sum()} of {status.size} corners kept, {(status == -1).sum()} moved; rms {np.sqrt((e ** 2).mean()):.4f} max {e.max():.4f} px")
    # cornerSubPix itself (equal to OpenCV's to 1e-3 px, tests/test_aprilgrid.py) sets this: measured on an H100, rms 0.073-0.079 px
    # and max 0.17-0.19 px; OpenCV's own cornerSubPix on the committed frames is 0.13 px off the truth at most
    assert kept.sum() >= 0.85 * status.size
    assert np.sqrt((e ** 2).mean()) <= 0.1 and e.max() <= 0.25


def test_blur_and_noise(api):
    img, truth, _ = _render("pinhole", 0.6, 20.0, 45.0, 10.0, blur_sigma_px=1.0, noise_sigma_dn=3.0)
    uv, status, found, _ = api.extract_aprilgrid(img, NX, NY)
    assert found[0]
    kept = status[0] == 1
    e = np.linalg.norm(uv[0][kept] - truth[kept], axis=1)
    print(f"blur 1 px, noise 3 DN: {kept.sum()} kept, rms {np.sqrt((e ** 2).mean()):.4f} max {e.max():.4f} px")
    assert kept.sum() >= 130 and e.max() < 0.3


def test_rule_fewer_than_four_tags(api):
    img3 = _render("pinhole", 0.3, nx=3, ny=1, tags_x=3, tags_y=1)[0]
    img4 = _render("pinhole", 0.3, nx=4, ny=1, tags_x=4, tags_y=1)[0]
    uv, status, found, s = api.extract_aprilgrid(np.stack([img3, img4]), 4, 1)
    assert found.tolist() == [False, True] and s["n_few_tags"] == 1, s
    assert (status[0] == 0).all() and np.isnan(uv[0]).all()
    assert (status[1] == 1).sum() >= 14


def test_rule_duplicate_id(api):
    ids = np.arange(NX * NY); ids[20] = 3
    uv, status, found, s = api.extract_aprilgrid(_render("pinhole", tag_ids=ids)[0], NX, NY)
    assert not found[0] and s["n_duplicate"] == 1 and (status == 0).all(), s


def test_rule_id_36_and_above(api):
    # ids 36 to 41 on a board of 6 x 7 = 42 tags: the wrapper drops them although the board has them
    ids = np.arange(42)
    img, truth, _ = _render("pinhole", 0.6, nx=6, ny=7, tags_x=6, tags_y=7, tag_ids=ids)
    uv, status, found, s = api.extract_aprilgrid(img, 6, 7)
    assert found[0] and s["n_id_range"] == 6, s
    assert (status[0, 4 * 36:] == 0).all() and (status[0, :4 * 36] == 1).sum() >= 130


def test_rule_border(api):
    # the board shifted so that the left column of tags is cut by the image border or lies within 4 px of it
    img, truth, valid = _render("pinhole", 0.5, offset=(0.23, 0.0))
    uv, status, found, s = api.extract_aprilgrid(img, NX, NY)
    assert found[0] and s["n_border"] >= 1, s
    for t in range(NX * NY):
        q = truth[4 * t:4 * t + 4]
        if (q[:, 0] < 3.5).any():
            assert (status[0, 4 * t:4 * t + 4] == 0).all(), t


def test_rule_displacement(api):
    # a second X-junction pasted 3 px right and 2 px down of a tag corner: cornerSubPix leaves for it, further than the radius
    img, truth, _ = _render("pinhole", 0.75)
    pid = (14 << 2) + 2
    x, y = np.rint(truth[pid]).astype(int)
    out = img.copy()
    out[y - 6 + 2:y + 6 + 2, x - 6 + 3:x + 6 + 3] = img[y - 6:y + 6, x - 6:x + 6]
    uv, status, found, s = api.extract_aprilgrid(np.stack([img, out]), NX, NY)
    print("displacement case:", status[:, pid], uv[:, pid], truth[pid], s["n_corners_moved"])
    assert found.all() and status[0, pid] == 1 and status[1, pid] == -1
    assert np.linalg.norm(uv[1, pid] - truth[pid]) > 2.0


def test_bit_identical_however_frames_arrive(api, golden):
    import torch
    imgs = np.concatenate([golden["frames"], np.stack([_render(n, 0.6, 20.0, 30.0, 40.0)[0] for n in CAMERAS])])
    ref = api.extract_aprilgrid(imgs, NX, NY)
    assert ref[2].sum() >= len(imgs) - 1

    def same(r):
        np.testing.assert_array_equal(r[0], ref[0]); np.testing.assert_array_equal(r[1], ref[1]); np.testing.assert_array_equal(r[2], ref[2])
    same(api.extract_aprilgrid(torch.from_numpy(imgs).cuda(), NX, NY))
    for chunk in ("1", "5"):
        os.environ["ICC_BOARD_CHUNK_FRAMES"] = chunk
        try:
            same(api.extract_aprilgrid(imgs, NX, NY))
        finally:
            del os.environ["ICC_BOARD_CHUNK_FRAMES"]
    pitched = np.zeros(imgs.shape[:2] + (imgs.shape[2] + 37,), dtype=np.uint8)
    pitched[:, :, :imgs.shape[2]] = imgs
    same(api.extract_aprilgrid(pitched[:, :, :imgs.shape[2]], NX, NY))
    same(api.extract_aprilgrid(torch.from_numpy(pitched).cuda()[:, :, :imgs.shape[2]], NX, NY))


def test_downsample(api, golden):
    uv1, st1, f1, _ = api.extract_aprilgrid(golden["frames"][:1], NX, NY, 1.0)
    uv2, st2, f2, s = api.extract_aprilgrid(golden["frames"][:1], NX, NY, 2.0)
    assert (s["width"], s["height"]) == (480, 270) and f1[0] and f2[0]
    both = (st1[0] == 1) & (st2[0] == 1)
    assert both.sum() >= 100
    assert np.abs((uv1[0][both] + 0.5) / 2 - 0.5 - uv2[0][both]).max() < 0.25


def test_corner_file_through_calibrate_camera_and_poses(tmp_path):
    name = "fisheye"
    model, intr = CAMERAS[name]
    rays = syn.camera_rays(model, intr, SIZE, 2)
    rng = np.random.default_rng(4)
    imgs = []
    for k in range(24):
        R, t = syn.aprilgrid_view_pose(NX, NY, S, rng.uniform(0.25, 0.4), rng.uniform(0, 40), rng.uniform(0, 360), rng.uniform(-30, 30),
                                       (rng.uniform(-0.08, 0.08), rng.uniform(-0.05, 0.05)))
        imgs.append(syn.render_aprilgrid(model, intr, SIZE, R, t, NX, NY, S, supersample=2, blur_sigma_px=0.6, noise_sigma_dn=1.5, seed=k, rays=rays)[0])
    ex = calibrator.AprilGridExtractor(S, NX, NY)
    path = tmp_path / "corners.uson"
    scene = ex.write(str(path), np.stack(imgs), 1.0 + np.arange(len(imgs)) / 30.0)
    assert io_formats.ubjson_loads(open(path, "rb").read()) == scene
    assert scene["calibration_board_type"] == 2 and len(scene["scene_pts"]) == 4 * NX * NY
    print("views:", len(scene["views"]), ex.summary)
    assert len(scene["views"]) >= 20
    out = tmp_path / "calib"
    r = subprocess.run([os.path.join(BIN, "calibrate_camera"), "--input_corners", str(path), "--camera_model_to_calibrate", "FISHEYE",
                        "--save_path_calib_dataset", str(out), "--grid_size=0"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    k = json.load(open(str(out) + ".json"))["intrinsics"]
    err = (k["focal_length"] - intr[0], k["principal_pt_x"] - intr[3], k["principal_pt_y"] - intr[4])
    print(f"fisheye: focal length error {err[0]:+.3f} px, principal point error ({err[1]:+.3f}, {err[2]:+.3f}) px")
    assert max(abs(e) for e in err) < 1.0, err
    poses = tmp_path / "poses.json"
    r = subprocess.run([os.path.join(BIN, "estimate_camera_poses_from_checkerboard"), "--input_corners=" + str(path), "--camera_calibration_json",
                        str(out) + ".json", "--output_pose_dataset=" + str(poses)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr + r.stdout
    assert len(json.load(open(poses))["views"]) >= 20
