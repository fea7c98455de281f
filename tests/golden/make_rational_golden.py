"""Reference pixels of OpenCV's rational polynomial model (CALIB_RATIONAL_MODEL) and of its fisheye module, computed by cv2.projectPoints /
cv2.fisheye.projectPoints themselves, for tests/test_rational.py.  Stored as tests/golden/rational_opencv_projectpoints.npz so that
no test needs cv2: per case the camera matrix K, the OpenCV coefficient vector D (k1, k2, p1, p2, k3, k4, k5, k6 / fisheye k1..k4), the
camera-frame points and OpenCV's pixels.  Skew is 0: cv2.projectPoints ignores K[0][1].
Run from the repo root:  python tests/golden/make_rational_golden.py
"""
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rational_opencv_projectpoints.npz")


def cases(seed=20261018):
    """(K, D, points) of the rational cases, then the fisheye case; points in front of the camera within each lens's field"""
    rng = np.random.default_rng(seed)
    out = []
    # typical wide-angle fits (k4..k6 carry most of the distortion), a near-pinhole one and one with large denominators
    Ds = [[0.35, -0.08, 1.2e-3, -8e-4, 0.004, 0.72, -0.02, 0.01],
          [-0.02, 0.01, -3e-4, 2e-4, -1e-3, 0.01, 0.002, -5e-4],
          [1.8, 0.9, 5e-4, 1e-3, 0.05, 2.1, 1.4, 0.2]]
    for D, half_fov in zip(Ds, (0.9, 0.6, 1.0)):
        fx = rng.uniform(400, 900); fy = fx * rng.uniform(0.98, 1.02)
        K = np.array([[fx, 0.0, rng.uniform(600, 680)], [0.0, fy, rng.uniform(330, 390)], [0.0, 0.0, 1.0]])
        n = 200
        ang = rng.uniform(0.0, half_fov, n); ph = rng.uniform(0, 2 * np.pi, n); dist = rng.uniform(0.3, 6.0, n)
        P = np.stack([np.tan(ang) * np.cos(ph), np.tan(ang) * np.sin(ph), np.ones(n)], -1) * (dist / np.sqrt(1 + np.tan(ang) ** 2))[:, None]
        out.append(("rational", K, np.array(D), P))
    fx = 380.0
    K = np.array([[fx, 0.0, 640.5], [0.0, fx * 1.003, 361.2], [0.0, 0.0, 1.0]])
    D = np.array([0.05, -0.012, 0.003, -4e-4])
    ang = rng.uniform(0.0, 1.45, 200); ph = rng.uniform(0, 2 * np.pi, 200)
    P = np.stack([np.sin(ang) * np.cos(ph), np.sin(ang) * np.sin(ph), np.cos(ang)], -1) * rng.uniform(0.3, 6.0, (200, 1))
    out.append(("fisheye", K, D, P))
    return out


def project(kind, K, D, P):
    import cv2
    if kind == "fisheye":
        uv, _ = cv2.fisheye.projectPoints(P.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, D)
    else:
        uv, _ = cv2.projectPoints(P, np.zeros(3), np.zeros(3), K, D)
    return uv.reshape(-1, 2)


def main():
    arrays = {}
    for i, (kind, K, D, P) in enumerate(cases()):
        arrays[f"kind_{i}"] = np.array(kind); arrays[f"K_{i}"] = K; arrays[f"D_{i}"] = D; arrays[f"points_{i}"] = P
        arrays[f"uv_{i}"] = project(kind, K, D, P)
    arrays["n_cases"] = np.array(len(cases()))
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
