"""Writes tests/golden/aprilgrid_opencv.npz: Kalibr AprilGrid frames drawn with OpenCV's own tag36h11 markers, what OpenCV's ArUco
detector finds in them, and cv2.cornerSubPix results under the AprilGrid wrapper's window rule.  Needs OpenCV >= 4.7 (cv2.aruco).

The board: 6 x 6 tags of side s with spacing 0.3 s, tag t = 6 y + x with its lower-left corner at (1.3 s x, 1.3 s y) in the board
frame (y up), and a black square of side 0.3 s in every gap crossing, the outer ones included (Kalibr's corner squares).  Each
tag is cv2.aruco.generateImageMarker(DICT_APRILTAG_36h11, t, borderBits=2) turned by 180 degrees, which is how the codes of
tag36h11 read on the printed board (DESIGN.md "AprilGrid corners").  Frames are 960 x 540 pinhole views, drawn by
cv2.warpPerspective at 4x and reduced with INTER_AREA.

Contents:
  frames (N, 540, 960) uint8, names (N,), truth (N, 144, 2) the board's corners in id order (t << 2) + i, i = bottom-left,
  bottom-right, top-right, top-left;
  cv_ids (M,), cv_frame (M,), cv_corners (M, 4, 2) OpenCV's detections (CORNER_REFINE_SUBPIX) in OpenCV's corner order;
  cv_refined (M, 4, 2), cv_moved (M, 4): those corners after cv2.cornerSubPix with the wrapper's window, and whether the wrapper's
  displacement rule drops them.  ArUco's own corners sit 1-2 px off the X-junctions that Kalibr's corner squares make (its
  contour runs round the squares' touching pixels), so the comparison is with the refined ones, which is the wrapper's order:
  detect, then cornerSubPix;
  bits (587, 6, 6) OpenCV's DICT_APRILTAG_36h11 bits;
  sp_frame (K,), sp_start (K, 2), sp_win (K,), sp_out (K, 2): cv2.cornerSubPix from the start points with window half-size sp_win.
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NX = NY = 6
S = 0.04
W, H = 960, 540
PPC = 24            # texture pixels per tag cell
SS = 4              # supersampling of the warp


def texture():
    """Board texture (rows from the board's top) and the texture coordinates of board point (x, y): pixel k spans [k - 0.5, k + 0.5]."""
    d = cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_APRILTAG_36h11)
    tag = 10 * PPC
    gap = int(round(0.3 * tag))
    pitch = tag + gap
    margin = 2 * tag
    side_x, side_y = NX * pitch - gap + 2 * margin, NY * pitch - gap + 2 * margin
    tex = np.full((side_y, side_x), 255, np.uint8)
    top = margin + NY * pitch - gap        # texture row of board y = 0 (an edge)

    def rows(y0, y1):                       # board y interval (texture units from the board's bottom) -> texture rows
        return top - y1, top - y0
    for ty in range(NY):
        for tx in range(NX):
            m = cv2.aruco.generateImageMarker(d, ty * NX + tx, tag, borderBits=2)
            r0, r1 = rows(ty * pitch, ty * pitch + tag)
            tex[r0:r1, margin + tx * pitch:margin + tx * pitch + tag] = np.rot90(m, 2)
    for ky in range(NY + 1):
        for kx in range(NX + 1):
            r0, r1 = rows(ky * pitch - gap, ky * pitch)
            c0 = margin + kx * pitch - gap
            tex[r0:r1, c0:c0 + gap] = 0
    scale = tag / S                          # texture px per metre

    def to_tex(xb, yb):
        return np.stack([margin - 0.5 + xb * scale, top - 0.5 - yb * scale], -1)
    return tex, to_tex, scale


def board_points():
    i = np.arange(NX * NY * 4)
    t, c = i >> 2, i & 3
    x = (t % NX) * S * 1.3 + np.array([0, S, S, 0])[c]
    y = (t // NX) * S * 1.3 + np.array([0, 0, S, S])[c]
    return np.stack([x, y, np.zeros_like(x)], -1)


def rot(axis, deg):
    a = np.deg2rad(deg)
    k = np.asarray(axis, float) / np.linalg.norm(axis)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx


K = np.array([[820.0, 0, 479.5], [0, 820.0, 269.5], [0, 0, 1]])


def pose(dist, tilt_axis=(0, 1, 0), tilt=0.0, roll=0.0, shift=(0.0, 0.0)):
    """Board-to-camera (R, t): the board upright (camera y = -board y) at `dist` in front of the board centre, tilted and rolled."""
    R0 = np.diag([1.0, -1.0, -1.0])
    R = rot((0, 0, 1), roll) @ rot(tilt_axis, tilt) @ R0
    c = np.array([(NX * 1.3 - 0.3) * S / 2, (NY * 1.3 - 0.3) * S / 2, 0.0])
    t = np.array([shift[0], shift[1], dist]) - R @ c
    return R, t


VIEWS = [  # name, pose, blur sigma (px), noise sigma (DN)
    ("frontal", pose(0.55), 0.0, 0.0),
    ("tilt_yaw", pose(0.6, (0, 1, 0), 35.0, 15.0), 0.0, 0.0),
    ("tilt_pitch_roll", pose(0.6, (1, 0, 0), 40.0, -70.0), 0.0, 0.0),
    ("upside_down", pose(0.6, (1, 1, 0), 20.0, 180.0), 0.0, 0.0),
    ("partial_right", pose(0.45, (0, 1, 0), 10.0, 5.0, shift=(0.2, 0.05)), 0.0, 0.0),
    ("close_partial", pose(0.3, (1, 0, 0), 15.0, 30.0, shift=(-0.05, 0.04)), 0.0, 0.0),
    ("blurred", pose(0.65, (1, 0, 0), 25.0, 100.0), 1.2, 0.0),
    ("noisy", pose(0.7, (0, 1, 0), -30.0, -20.0), 0.0, 3.0),
]


def render(tex, to_tex, R, t, blur, noise, seed):
    # homography from texture pixels to the supersampled image: x_img ~ K [r1 r2 t] B^-1 x_tex
    pts = np.array([[0, 0], [1, 0], [0, 1]], float)
    tp = to_tex(pts[:, 0], pts[:, 1])
    A = np.array([[tp[1, 0] - tp[0, 0], tp[2, 0] - tp[0, 0], tp[0, 0]], [tp[1, 1] - tp[0, 1], tp[2, 1] - tp[0, 1], tp[0, 1]], [0, 0, 1]])
    Hb = K @ np.column_stack([R[:, 0], R[:, 1], t])          # board (x, y, 1) -> image
    Hs = np.diag([SS, SS, 1.0]) @ np.array([[1, 0, 0.5], [0, 1, 0.5], [0, 0, 1]]) @ Hb @ np.linalg.inv(A)
    Hs = np.array([[1, 0, -0.5], [0, 1, -0.5], [0, 0, 1]]) @ Hs   # image (pixel centres at integers) -> supersampled pixel centres
    big = cv2.warpPerspective(tex, Hs, (W * SS, H * SS), flags=cv2.INTER_LINEAR, borderValue=255)
    img = cv2.resize(big, (W, H), interpolation=cv2.INTER_AREA).astype(np.float64)
    img = 25.0 + (225.0 - 25.0) * img / 255.0
    if blur > 0:
        img = cv2.GaussianBlur(img, (0, 0), blur)
    if noise > 0:
        img = img + np.random.default_rng(seed).normal(0.0, noise, img.shape)
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    pc = board_points() @ R.T + t
    uv = pc @ K.T
    return img, uv[:, :2] / uv[:, 2:]


def window(q):
    """The wrapper's displacement limit r = max(2, 0.075 perimeter / 4 - 1) and window half-size ceil(r + 1) for a tag's corners."""
    per = float(np.sum(np.linalg.norm(q.astype(np.float64) - np.roll(q, -1, 0), axis=1)))
    r = max(2.0, 0.075 * per / 4 - 1.0)
    return r, int(np.ceil(r + 1.0))


def main():
    tex, to_tex, _ = texture()
    d = cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_APRILTAG_36h11)
    p = cv2.aruco.DetectorParameters()
    p.markerBorderBits = 2
    p.cornerRefinementMethod = cv2.aruco.CORNER_REFINE_SUBPIX
    # a fixed 9 x 9 window: the default, relative to the marker, reaches the far corners of the corner squares on large tags
    p.cornerRefinementWinSize = 4
    p.relativeCornerRefinmentWinSize = 0.0
    det = cv2.aruco.ArucoDetector(d, p)
    frames, truth, names = [], [], []
    cv_ids, cv_frame, cv_corners, cv_refined, cv_moved = [], [], [], [], []
    sp_frame, sp_start, sp_win, sp_out = [], [], [], []
    rng = np.random.default_rng(42)
    crit = (cv2.TERM_CRITERIA_EPS + cv2.TERM_CRITERIA_MAX_ITER, 100, 0.01)
    for k, (name, (R, t), blur, noise) in enumerate(VIEWS):
        img, uv = render(tex, to_tex, R, t, blur, noise, seed=k)
        frames.append(img); truth.append(uv); names.append(name)
        corners, ids, _ = det.detectMarkers(img)
        ids = [] if ids is None else ids.ravel().tolist()
        for c, i in zip(corners, ids):
            c = c.reshape(4, 2)
            r, win = window(c)
            ref = cv2.cornerSubPix(img, c.copy(), (win, win), (-1, -1), crit)
            cv_ids.append(i); cv_frame.append(k); cv_corners.append(c); cv_refined.append(ref)
            cv_moved.append(np.sum((ref.astype(np.float64) - c) ** 2, axis=1) > r * r)
        # cornerSubPix from perturbed true corners of every tag well inside the frame, window from the tag's perimeter
        for tg in range(NX * NY):
            q = uv[4 * tg:4 * tg + 4]
            if (q < 12).any() or (q[:, 0] > W - 13).any() or (q[:, 1] > H - 13).any():
                continue
            _, win = window(q)
            start = (q + rng.uniform(-1.2, 1.2, q.shape)).astype(np.float32)
            out = cv2.cornerSubPix(img, start.copy(), (win, win), (-1, -1), crit)
            for j in range(4):
                sp_frame.append(k); sp_start.append(start[j]); sp_win.append(win); sp_out.append(out[j])
    bits = np.stack([cv2.aruco.Dictionary.getBitsFromByteList(d.bytesList[i:i + 1, 0], 6) for i in range(d.bytesList.shape[0])])
    np.savez_compressed(os.path.join(HERE, "aprilgrid_opencv.npz"), frames=np.stack(frames), names=np.array(names), truth=np.stack(truth),
                        cv_ids=np.array(cv_ids, np.int32), cv_frame=np.array(cv_frame, np.int32), cv_corners=np.array(cv_corners, np.float32),
                        cv_refined=np.array(cv_refined, np.float32), cv_moved=np.array(cv_moved, bool),
                        bits=bits.astype(np.uint8), sp_frame=np.array(sp_frame, np.int32), sp_start=np.array(sp_start, np.float32),
                        sp_win=np.array(sp_win, np.int32), sp_out=np.array(sp_out, np.float32), opencv_version=np.array(cv2.__version__))
    for k, n in enumerate(names):
        print(n, "opencv tags:", sum(1 for f in cv_frame if f == k))


if __name__ == "__main__":
    main()
