"""Writes tests/golden/radon_board_opencv.npz: radon-board frames from synthetic.render_radon_board, what OpenCV's
findChessboardCornersSBWithMeta returns for them (the overload BoardExtractor calls) with the reference's flags (BoardExtractor::InitializeRadonBoard:
CALIB_CB_LARGER | CALIB_CB_MARKER | CALIB_CB_EXHAUSTIVE), and cv2.resize(INTER_LINEAR) of the first frame at several factors.

Run once where cv2 is importable (python tests/golden/make_radon_golden.py); no test imports cv2.
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from openimucameracalibrator_b200 import camera_models as cm, synthetic as syn  # noqa: E402

SIZE = (640, 480)
W, H, SQ = 14, 9, 0.03
PINHOLE = (cm.PINHOLE, (600.0, 1.0, 0.0, 320.0, 240.0, -0.05, 0.01))
FISHEYE = (cm.FISHEYE, (300.0, 1.0, 0.0, 318.0, 242.0, 0.05, 0.07, -0.11, 0.05))
# (name, camera, distance, tilt, tilt axis, roll, board offset)
FRAMES = [
    ("pinhole", PINHOLE, 0.9, 25.0, 30.0, 0.0, (0.0, 0.0)),
    ("fisheye", FISHEYE, 0.45, 35.0, 120.0, 10.0, (0.0, 0.0)),
    ("pinhole_roll90", PINHOLE, 1.1, 20.0, 200.0, 90.0, (0.0, 0.0)),
    ("pinhole_roll180", PINHOLE, 0.9, 30.0, 80.0, 180.0, (0.0, 0.0)),
    ("no_board", PINHOLE, 0.9, 0.0, 0.0, 0.0, (5.0, 0.0)),
    ("cut_by_border", PINHOLE, 0.8, 15.0, 0.0, 0.0, (0.36, 0.0)),
]
FACTORS = (2.0, 1.5, 3.0)
FLAGS = cv2.CALIB_CB_LARGER | cv2.CALIB_CB_MARKER | cv2.CALIB_CB_EXHAUSTIVE


def main():
    imgs, found, corners, truth, truth_valid = [], [], [], [], []
    for name, (model, intr), dist, tilt, axis, roll, off in FRAMES:
        R, t = syn.radon_view_pose(W, H, SQ, dist, tilt, axis, roll, off)
        img, uv, valid = syn.render_radon_board(model, intr, SIZE, R, t, W, H, SQ, blur_sigma_px=0.6)
        ok, c, _ = cv2.findChessboardCornersSBWithMeta(img, (W, H), FLAGS)
        imgs.append(img); found.append(bool(ok)); truth.append(uv); truth_valid.append(valid)
        corners.append(c.reshape(-1, 2).astype(np.float64) if ok else np.full((W * H, 2), np.nan))
        print(name, "found" if ok else "not found")
    odd = imgs[0][:479, :639]   # odd height and width: INTER_AREA's border block at scale 2
    resized = {"resize_odd_2": cv2.resize(odd, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_LINEAR),
               "resize_odd_1p5": cv2.resize(odd, None, fx=1 / 1.5, fy=1 / 1.5, interpolation=cv2.INTER_LINEAR)}
    resized.update({f"resize_{f:g}".replace(".", "p"): cv2.resize(imgs[0], None, fx=1.0 / f, fy=1.0 / f, interpolation=cv2.INTER_LINEAR) for f in FACTORS})
    np.savez_compressed(os.path.join(HERE, "radon_board_opencv.npz"), names=np.array([f[0] for f in FRAMES]), models=np.array([f[1][0] for f in FRAMES]),
                        frames=np.stack(imgs), found=np.array(found), corners=np.stack(corners), truth=np.stack(truth), truth_valid=np.stack(truth_valid),
                        corners_x=W, corners_y=H, factors=np.array(FACTORS), opencv_version=cv2.__version__, **resized)


if __name__ == "__main__":
    main()
