"""Radon checkerboard extraction without a GPU: the product's downsample, response and sub-pixel step (csrc/icc_board_math.cuh,
compiled for the CPU from tests/board/board_host_math.cu) against NumPy statements of the same rules and against committed
cv2.resize output; the renderer's board layout; the C-ABI's argument checks."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from openimucameracalibrator_b200 import synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_board_"), "libboard_host_math.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "board", "board_host_math.cu")])
        _LIB = ctypes.CDLL(out)
        _LIB.bm_resize.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_void_p]
        _LIB.bm_resize_dim.argtypes = [ctypes.c_int, ctypes.c_double]
        _LIB.bm_response.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        _LIB.bm_refine.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_float, ctypes.c_void_p]
        _LIB.bm_half_window.argtypes = [ctypes.c_float]
        _LIB.bm_subpix_step.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int, ctypes.c_void_p]
    return _LIB


def product_resize(img, f):
    img = np.ascontiguousarray(img)
    h, w = img.shape
    dw, dh = lib().bm_resize_dim(w, f), lib().bm_resize_dim(h, f)
    out = np.zeros((dh, dw), np.uint8)
    lib().bm_resize(img.ctypes.data, w, w, h, float(f), out.ctypes.data)
    return out


def numpy_resize(img, f):
    """cv::resize(INTER_LINEAR) on 8-bit gray as OpenCV computes it: exactly scale 2 is INTER_AREA's 2x2 mean with +2 >> 2, any other
    scale 11-bit fixed-point bilinear weights from float source coordinates, then ((b0 (S0 >> 4)) >> 16) + ((b1 (S1 >> 4)) >> 16) + 2) >> 2."""
    sh, sw = img.shape
    dw, dh = int(np.rint(sw / f)), int(np.rint(sh / f))
    scale = 1.0 / (1.0 / f)
    I = img.astype(np.int64)
    if scale == 2.0:
        a = I[:2 * dh, :2 * dw]
        return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)

    def coeff(n, ssize, clamp_hi):
        fx = ((np.arange(n) + 0.5) * scale - 0.5).astype(np.float32)
        s = np.floor(fx).astype(np.int64)
        fx = (fx - s.astype(np.float32)).astype(np.float32)
        fx[s < 0] = 0; s[s < 0] = 0
        if clamp_hi:
            hi = s >= ssize - 1
            fx[hi] = 0; s[hi] = ssize - 1
        return s, np.rint((np.float32(1) - fx) * np.float32(2048)).astype(np.int64), np.rint(fx * np.float32(2048)).astype(np.int64)
    sx, a0, a1 = coeff(dw, sw, True)
    sy, b0, b1 = coeff(dh, sh, False)
    S = I[:, sx] * a0 + I[:, np.minimum(sx + 1, sw - 1)] * a1
    S0, S1 = S[np.clip(sy, 0, sh - 1)], S[np.clip(sy + 1, 0, sh - 1)]
    return ((((b0[:, None] * (S0 >> 4)) >> 16) + ((b1[:, None] * (S1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)


def numpy_response(img):
    """3x3 box mean, then (max - min)^2 / 81 of the four 9-pixel line sums at 0, 45, 90 and 135 degrees; 0 within 5 px of the border."""
    h, w = img.shape
    I = img.astype(np.float64)
    B = np.zeros((h, w))
    B[1:-1, 1:-1] = sum(I[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx] for dy in (-1, 0, 1) for dx in (-1, 0, 1)) / 9.0
    R = 4
    ys, xs = np.mgrid[R + 1:h - R - 1, R + 1:w - R - 1]
    L = [sum(B[ys + t * dy, xs + t * dx] for t in range(-R, R + 1)) for dx, dy in ((1, 0), (1, 1), (0, 1), (-1, 1))]
    out = np.zeros((h, w))
    out[R + 1:h - R - 1, R + 1:w - R - 1] = ((np.max(L, 0) - np.min(L, 0)) / 9.0) ** 2
    return out


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "radon_board_opencv.npz"))


def test_downsample_equals_committed_cv2_resize(golden):
    for f in golden["factors"]:
        ref = golden["resize_" + f"{f:g}".replace(".", "p")]
        np.testing.assert_array_equal(product_resize(golden["frames"][0], f), ref)
    odd = golden["frames"][0][:479, :639]   # odd sizes: INTER_AREA's border block at scale 2
    np.testing.assert_array_equal(product_resize(odd, 2.0), golden["resize_odd_2"])
    np.testing.assert_array_equal(product_resize(odd, 1.5), golden["resize_odd_1p5"])


@pytest.mark.parametrize("f", [1.25, 1.5, 2.0, 2.5, 3.0, 4.0, 1.0 / 0.3])
def test_downsample_equals_numpy_statement(f):
    img = np.random.default_rng(3).integers(0, 256, (122, 206), dtype=np.uint8)
    np.testing.assert_array_equal(product_resize(img, f), numpy_resize(img, f))


def test_response_equals_numpy_statement(golden):
    img = np.ascontiguousarray(golden["frames"][1][100:220, 200:380])
    h, w = img.shape
    box, resp = np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
    lib().bm_response(img.ctypes.data, w, h, box.ctypes.data, resp.ctypes.data)
    ref = numpy_response(img)
    assert np.abs(resp - ref).max() <= 1e-5 * ref.max()
    # the response peaks at the board's corners: every local maximum above 0.4 of the largest lies within 2.5 px of a true corner
    # (the response is flat within about a pixel of an X-junction; the sub-pixel step starts from there)
    tr = golden["truth"][1] - [200, 100]
    from scipy.ndimage import maximum_filter
    pk = np.argwhere((resp == maximum_filter(resp, 7)) & (resp >= 0.4 * resp.max()))
    d = np.min(np.hypot(tr[:, 0][None] - pk[:, 1][:, None], tr[:, 1][None] - pk[:, 0][:, None]), axis=1)
    assert len(pk) > 10 and d.max() <= 2.5


def numpy_subpix_step(I, qx, qy, hw):
    """One gradient-orthogonality step at q: the pixels round(q) +- (hw + hw // 2) whose central differences stay in the image, Gaussian weights
    exp(-|p - q|^2 / (2 (hw / 2)^2)), and the 2x2 solve of (sum w g g^T) q' = sum w g g^T p."""
    I = np.asarray(I, dtype=np.float64)
    h, w = I.shape
    cx, cy = int(np.floor(qx + 0.5)), int(np.floor(qy + 0.5))
    r = hw + hw // 2
    py, px = np.mgrid[cy - r:cy + r + 1, cx - r:cx + r + 1]
    ok = (px >= 1) & (py >= 1) & (px <= w - 2) & (py <= h - 2)
    px, py = px[ok], py[ok]
    gx, gy = 0.5 * (I[py, px + 1] - I[py, px - 1]), 0.5 * (I[py + 1, px] - I[py - 1, px])
    wt = np.exp(-((px - qx) ** 2 + (py - qy) ** 2) * 2.0 / hw ** 2)
    A = np.array([[np.sum(wt * gx * gx), np.sum(wt * gx * gy)], [np.sum(wt * gx * gy), np.sum(wt * gy * gy)]])
    b = np.array([np.sum(wt * (gx * gx * px + gx * gy * py)), np.sum(wt * (gx * gy * px + gy * gy * py))])
    return np.linalg.solve(A, b)


def _saddle(w, h, cx, cy, angle, sigma=1.0, amp=110.0):
    """A Gaussian-blurred X-junction at (cx, cy), exactly: sign(u) sign(v) in the frame rotated by `angle`, blurred, is
    erf(u / (sigma sqrt 2)) erf(v / (sigma sqrt 2)), sampled at the pixel centres (float, not quantised)."""
    from scipy.special import erf
    X, Y = np.meshgrid(np.arange(w) - cx, np.arange(h) - cy)
    c, s = np.cos(angle), np.sin(angle)
    return 125.0 + amp * erf((c * X + s * Y) / (sigma * np.sqrt(2))) * erf((-s * X + c * Y) / (sigma * np.sqrt(2)))


SADDLES = [(30.3, 29.6, 0.3), (31.77, 30.21, 1.0), (30.13, 30.41, 0.0), (29.5, 30.5, -0.6)]


@pytest.mark.parametrize("cx,cy,angle", SADDLES)
def test_subpixel_step_equals_numpy_statement(cx, cy, angle):
    img = np.rint(_saddle(64, 60, cx, cy, angle)).astype(np.uint8)
    for q, hw in (((round(cx) + 1.0, round(cy) - 1.0), 8), ((cx + 0.3, cy - 0.2), 4), ((cx - 3.4, cy + 2.2), 5)):
        out = np.zeros(2)
        assert lib().bm_subpix_step(img.ctypes.data, 64, 60, q[0], q[1], hw, out.ctypes.data) == 1
        np.testing.assert_allclose(out, numpy_subpix_step(img, q[0], q[1], hw), rtol=0, atol=1e-9)


@pytest.mark.parametrize("cx,cy,angle", SADDLES)
def test_subpixel_refinement_converges_to_saddle(cx, cy, angle):
    # the rule itself, on the exact (unquantised) saddle, converges to the analytic corner within 1e-3 px
    q = np.array([round(cx) + 1.0, round(cy) - 1.0])
    for _ in range(60):
        n = numpy_subpix_step(_saddle(64, 60, cx, cy, angle), q[0], q[1], 8)
        step, q = np.hypot(*(n - q)), n
        if step < 1e-9:
            break
    assert np.hypot(q[0] - cx, q[1] - cy) <= 1e-3
    # the product on the 8-bit image: rounding to whole grey levels moves the fixed point.  Along an axis-aligned edge every pixel
    # rounds the same way, so the rounding does not average out; measured 0.2e-3 .. 4.7e-3 px on these four saddles
    img = np.rint(_saddle(64, 60, cx, cy, angle)).astype(np.uint8)
    out = np.zeros(2)
    it = lib().bm_refine(img.ctypes.data, 64, 60, round(cx) + 1.0, round(cy) - 1.0, 24.0, out.ctypes.data)
    assert lib().bm_half_window(24.0) == 8 and 0 < it < 40
    assert np.hypot(out[0] - cx, out[1] - cy) <= 5e-3


def test_renderer_layout_matches_the_printed_board():
    # the vertex marker sits in a white square with a black dot, the arms in black squares with white dots, next to the centre
    W, H, s = 14, 9, 1.0
    mi, mj = syn.radon_marker_cell(W, H)
    assert (mi, mj) == (3, 6)
    shade = lambda i, j: syn.radon_board_shade(np.array([i * s]), np.array([j * s]), W, H, s)[0]  # noqa: E731
    assert shade(mi + 0.5, mj + 0.5) == 0.0 and shade(mi + 0.5 + 0.3, mj + 0.5 + 0.3) == 1.0
    assert shade(mi + 1.5, mj + 0.5) == 1.0 and shade(mi + 1.5 + 0.3, mj + 0.5 + 0.3) == 0.0
    assert shade(mi + 0.5, mj + 1.5) == 1.0 and shade(mi + 0.5 + 0.3, mj + 1.5 + 0.3) == 0.0
    # the printed top-left square is white, the bottom-left black; black border squares are rounded outward
    assert shade(H - 0.5, -0.5) == 1.0 and shade(-0.5, -0.5) == 0.0
    assert shade(H - 0.5 + 0.45, 0.5 - 0.45) == 1.0 and shade(H - 0.5, 0.5) == 0.0
    pts = syn.radon_board_points(W, H, 0.02)
    assert pts.shape == (W * H, 3) and np.allclose(pts[W + 2], [0.02, 0.04, 0.0])


def test_capi_rejects_bad_arguments_without_a_device():
    from openimucameracalibrator_b200 import calibrator
    lib_ = calibrator.load_library()
    h = ctypes.c_void_p()
    lib_.icc_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
    st = lib_.icc_create(ctypes.byref(h), -1)   # host-only handle
    if st != 0:
        pytest.skip("this build cannot create a host-only handle")
    f = lib_.icc_extract_radon_board
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    img = np.zeros((2, 40, 50), np.uint8); uv = np.zeros(2 * 14 * 9 * 2); found = np.zeros(2, np.int32)
    ok = (h, 2, 50, 40, 50, img.ctypes.data, 14, 9, 1.0, uv.ctypes.data, found.ctypes.data, None)
    bad = [dict(i=6, v=2), dict(i=7, v=2), dict(i=8, v=0.5), dict(i=8, v=float("nan")), dict(i=8, v=float("inf")), dict(i=4, v=49),
           dict(i=9, v=None), dict(i=10, v=None), dict(i=5, v=None)]
    for b in bad:
        args = list(ok); args[b["i"]] = b["v"]
        assert f(*args) == 1, b        # ICC_ERR_INVALID_ARGUMENT
    assert f(*ok) == 2                 # ICC_ERR_NO_DEVICE
    lib_.icc_destroy.argtypes = [ctypes.c_void_p]
    lib_.icc_destroy(h)
