"""Reference pixels for FISHEYE_RADIAL_TANGENTIAL (Kannala-Brandt with k1..k6 and tangential t1, t2), computed by OpenCV itself, for
tests/test_fisheye_radtan.py.  Stored as tests/golden/fisheye_radtan_opencv.npz so that no test needs cv2.  Two kinds of case:
  * "fisheye": the whole model with k5 = k6 = t1 = t2 = 0 is OpenCV's fisheye model, so cv2.fisheye.projectPoints gives its pixels,
    for rays up to 88 degrees off the axis;
  * "tangential": the radial stage (xr, yr) = (theta_d / r) (x, y) with all six radial terms, evaluated here in NumPy, then OpenCV's
    pinhole with distortion (0, 0, t1, t2, 0) applied to (xr, yr, 1), which is this model's tangential stage and affine (t1, t2 = p1, p2).
Per case: K, the radial terms k1..k6, the tangential terms (t1, t2), the camera-frame points, the radial-stage points fed to OpenCV and
OpenCV's pixels.  Skew is 0: cv2.projectPoints ignores K[0][1].
Run from the repo root:  python tests/golden/make_fisheye_radtan_golden.py
"""
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "fisheye_radtan_opencv.npz")


def _rays(rng, max_deg, n, min_deg=0.0):
    ang = np.radians(rng.uniform(min_deg, max_deg, n)); ph = rng.uniform(0, 2 * np.pi, n)
    return np.stack([np.sin(ang) * np.cos(ph), np.sin(ang) * np.sin(ph), np.cos(ang)], -1) * rng.uniform(0.3, 6.0, (n, 1))


def radial_stage(k16, P):
    """(xr, yr) = (theta_d / r) (x, y), theta_d = theta (1 + k1 theta^2 + ... + k6 theta^12), theta = atan2(r, z)"""
    r = np.hypot(P[:, 0], P[:, 1])
    th = np.arctan2(r, P[:, 2]); t = th * th
    c = np.asarray(k16, dtype=np.float64)
    poly = 1.0 + t * (c[0] + t * (c[1] + t * (c[2] + t * (c[3] + t * (c[4] + t * c[5])))))
    return P[:, :2] * (th * poly / r)[:, None]


def cases(seed=20261019):
    """(kind, K, k1..k6, (t1, t2), points): two fisheye cases (one with a ring of rays at 80..88 degrees), then three decentred lenses"""
    rng = np.random.default_rng(seed)
    out = []
    for D, max_deg in (([0.05, -0.012, 0.003, -4e-4], 88.0), ([-0.03, 0.004, -1e-3, 2e-4], 88.0)):
        fx = rng.uniform(300, 450)
        K = np.array([[fx, 0.0, rng.uniform(620, 660)], [0.0, fx * rng.uniform(0.99, 1.01), rng.uniform(340, 380)], [0.0, 0.0, 1.0]])
        P = np.concatenate([_rays(rng, max_deg, 200), _rays(rng, 88.0, 40, min_deg=80.0)])
        out.append(("fisheye", K, np.array(D + [0.0, 0.0]), np.zeros(2), P))
    for D, T, max_deg in (([0.05, -0.012, 0.003, -4e-4, 6e-5, -4e-6], [1.2e-3, -8e-4], 85.0),
                          ([-0.02, 0.01, -2e-3, 3e-4, -2e-5, 1e-6], [-5e-4, 2e-3], 85.0),
                          ([0.12, -0.05, 0.01, -1e-3, 5e-5, -1e-6], [3e-3, 1e-3], 70.0)):
        fx = rng.uniform(300, 450)
        K = np.array([[fx, 0.0, rng.uniform(620, 660)], [0.0, fx * rng.uniform(0.99, 1.01), rng.uniform(340, 380)], [0.0, 0.0, 1.0]])
        out.append(("tangential", K, np.array(D), np.array(T), _rays(rng, max_deg, 240)))
    return out


def project(kind, K, D, T, P):
    """OpenCV's pixels of the case, and the radial-stage points handed to cv2.projectPoints (the tangential kind only)"""
    import cv2
    if kind == "fisheye":
        uv, _ = cv2.fisheye.projectPoints(P.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, D[:4])
        return uv.reshape(-1, 2), np.zeros((0, 2))
    xr = radial_stage(D, P)
    X = np.concatenate([xr, np.ones((xr.shape[0], 1))], 1)
    uv, _ = cv2.projectPoints(X, np.zeros(3), np.zeros(3), K, np.array([0.0, 0.0, T[0], T[1], 0.0]))
    return uv.reshape(-1, 2), xr


def main():
    arrays = {}
    cs = cases()
    for i, (kind, K, D, T, P) in enumerate(cs):
        uv, xr = project(kind, K, D, T, P)
        arrays[f"kind_{i}"] = np.array(kind); arrays[f"K_{i}"] = K; arrays[f"D_{i}"] = D; arrays[f"T_{i}"] = T; arrays[f"points_{i}"] = P
        arrays[f"xr_{i}"] = xr; arrays[f"uv_{i}"] = uv
    arrays["n_cases"] = np.array(len(cs))
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
