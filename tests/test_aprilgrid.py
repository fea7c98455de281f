"""AprilGrid extraction without a GPU: the tag36h11 codebook against OpenCV's, the product's tag sampler and decoder and its
cornerSubPix (csrc/icc_aprilgrid_math.cuh, compiled for the CPU from tests/board/aprilgrid_host_math.cu) against ideal tags and
cv2.cornerSubPix, the wrapper's rules, the corner file's board points and the C-ABI's argument checks."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from openimucameracalibrator_b200 import calibrator, synthetic as syn

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_aprilgrid_"), "libaprilgrid_host_math.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "board", "aprilgrid_host_math.cu")])
        L = ctypes.CDLL(out)
        L.ag_code.restype = ctypes.c_uint64
        L.ag_rotate90.restype = ctypes.c_uint64
        L.ag_rotate90.argtypes = [ctypes.c_uint64]
        L.ag_decode.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.ag_corner_subpix.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
        L.ag_subpix_radius.restype = ctypes.c_double
        L.ag_subpix_radius.argtypes = [ctypes.c_double]
        L.ag_subpix_half_window.argtypes = [ctypes.c_double]
        L.ag_drop_reason.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ag_frame_verdict.argtypes = [ctypes.c_int, ctypes.c_void_p]
        _LIB = L
    return _LIB


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "aprilgrid_opencv.npz"))


def codes():
    return [int(lib().ag_code(i)) for i in range(lib().ag_code_count())]


def test_codebook_is_opencv_rotated_by_180_degrees(golden):
    c = codes()
    assert len(c) == 587 and len(set(c)) == 587 and max(c) < 1 << 36
    assert [int(x) for x in syn.tag36h11_codes()] == c            # the renderer reads the same header
    for i, b in enumerate(golden["bits"]):
        v = 0
        for bit in np.rot90(b, 2).ravel():
            v = (v << 1) | int(bit)
        assert v == c[i], i


def test_codebook_minimum_hamming_distance_over_rotations():
    c = np.array(codes(), dtype=np.uint64)
    rots = [c]
    for _ in range(3):
        rots.append(np.array([lib().ag_rotate90(int(x)) for x in rots[-1]], dtype=np.uint64))
    assert (np.array([lib().ag_rotate90(int(x)) for x in rots[3]], dtype=np.uint64) == c).all()   # four turns are the identity
    popc = np.vectorize(lambda x: bin(int(x)).count("1"))
    best = 36
    for k, r in enumerate(rots):
        d = popc(r[:, None] ^ c[None, :])
        if k == 0:
            np.fill_diagonal(d, 36)
        best = min(best, int(d.min()))
    assert best == 11


def printed_tag(code, flip=()):
    """10 x 10 cells of a tag as printed (rows from the top), 1 white; `flip` inverts data bits k (reading order)."""
    P = np.zeros((10, 10), np.uint8)
    for k in range(36):
        bit = (code >> (35 - k)) & 1
        if k in flip:
            bit ^= 1
        P[2 + k // 6, 2 + k % 6] = bit
    return P


def tag_image(cells, px=12, margin=40):
    """An axis-aligned tag of px-pixel cells on white, dark 30 and light 220, and its corners in the quad frame's order."""
    side = 10 * px
    img = np.full((side + 2 * margin, side + 2 * margin), 220, np.uint8)
    img[margin:margin + side, margin:margin + side] = np.where(np.kron(cells, np.ones((px, px), np.uint8)) == 1, 220, 30)
    a, b = margin - 0.5, margin + side - 0.5
    return img, np.array([a, b, b, b, b, a, a, a], float)   # bottom-left, bottom-right, top-right, top-left on screen


def decode(img, q):
    out = np.zeros(4, np.int32)
    code = ctypes.c_uint64()
    img = np.ascontiguousarray(img)
    lib().ag_decode(img.ctypes.data, img.shape[1], img.shape[0], q.ctypes.data, out.ctypes.data, ctypes.byref(code))
    return out, code.value


@pytest.mark.parametrize("tag_id", [0, 7, 35, 36, 586])
@pytest.mark.parametrize("turns", [0, 1, 2, 3])
def test_decoder_reads_ideal_tags_in_every_rotation(tag_id, turns):
    c = codes()[tag_id]
    img, q = tag_image(np.rot90(printed_tag(c), turns))
    out, code = decode(img, q)
    assert out[3] == 1 and (out[0], out[1]) == (tag_id, 0), (out, hex(code))
    # the decoded bottom-left is q[rot]: a quarter turn counter-clockwise on screen puts it at the bottom-right, q1
    assert out[2] == turns
    if turns == 0:
        assert code == c


@pytest.mark.parametrize("turns", [0, 1, 2, 3])
def test_decoder_corrects_one_bit_and_rejects_two(turns):
    for tag_id, flips in ((3, (0,)), (100, (17,)), (35, (35,))):
        out, _ = decode(*tag_image(np.rot90(printed_tag(codes()[tag_id], flips), turns)))
        assert (out[0], out[1], out[2]) == (tag_id, 1, turns)
        p = np.array([50.0, 50, 100, 50, 100, 100, 50, 100])
        assert lib().ag_drop_reason(p.ctypes.data, int(out[1]), int(out[0]), 400, 400) == (0 if tag_id < 36 else 3)
    for tag_id, flips in ((3, (0, 1)), (200, (5, 30))):
        out, _ = decode(*tag_image(np.rot90(printed_tag(codes()[tag_id], flips), turns)))
        assert out[1] >= 2
        p = np.array([50.0, 50, 100, 50, 100, 100, 50, 100])
        assert lib().ag_drop_reason(p.ctypes.data, int(out[1]), int(out[0]), 400, 400) == 2     # not good


def test_decoder_on_a_projected_tag():
    # a tag seen under perspective: sampling goes through the quad's projective map, not an affine one
    c = codes()[21]
    cells = printed_tag(c)
    H = np.array([[1.1, 0.25, 60.0], [-0.12, 0.95, 70.0], [0.0009, 0.0006, 1.0]])
    size = 320
    yy, xx = np.mgrid[0:size * 4, 0:size * 4]
    pts = np.stack([(xx + 0.5) / 4 - 0.5, (yy + 0.5) / 4 - 0.5, np.ones_like(xx, float)], -1) @ np.linalg.inv(H).T
    u, v = pts[..., 0] / pts[..., 2], pts[..., 1] / pts[..., 2]            # tag coordinates, 0..120 across, rows from the top
    inside = (u >= 0) & (u < 120) & (v >= 0) & (v < 120)
    val = np.where(inside, cells[np.clip(v // 12, 0, 9).astype(int), np.clip(u // 12, 0, 9).astype(int)], 1)
    img = np.rint(30 + 190 * val.reshape(size, 4, size, 4).mean(axis=(1, 3))).astype(np.uint8)
    corners = np.array([[0, 120], [120, 120], [120, 0], [0, 0]], float)
    cp = np.c_[corners, np.ones(4)] @ H.T
    q = (cp[:, :2] / cp[:, 2:]).ravel()
    out, _ = decode(img, q)
    assert (out[0], out[1], out[2], out[3]) == (21, 0, 0, 1)


def test_corner_subpix_matches_opencv(golden):
    frames = golden["frames"]
    out = np.zeros(2, np.float32)
    worst = 0.0
    for f, s, win, ref in zip(golden["sp_frame"], golden["sp_start"], golden["sp_win"], golden["sp_out"]):
        img = np.ascontiguousarray(frames[f])
        lib().ag_corner_subpix(img.ctypes.data, img.shape[1], img.shape[0], float(s[0]), float(s[1]), int(win), out.ctypes.data)
        worst = max(worst, float(np.abs(out - ref).max()))
    print(f"cornerSubPix: {len(golden['sp_win'])} corners, max |product - cv2| {worst:.2e} px")
    assert worst <= 1e-3


def test_window_rule():
    for per, r in ((40.0, 2.0), (100.0, 2.0), (160.0, 2.0), (400.0, 6.5), (1000.0, 17.75)):
        assert lib().ag_subpix_radius(per) == pytest.approx(r)
        assert lib().ag_subpix_half_window(r) == int(np.ceil(r + 1))


def test_wrapper_rules():
    def drop(p, ham=0, tag_id=0, w=100, h=80):
        p = np.asarray(p, float).ravel()
        return lib().ag_drop_reason(p.ctypes.data, ham, tag_id, w, h)
    ok = [[10, 10], [50, 10], [50, 50], [10, 50]]
    assert drop(ok) == 0
    assert drop([[3.99, 10], [50, 10], [50, 50], [10, 50]]) == 1                 # x < 4
    assert drop([[4.0, 10], [50, 10], [50, 50], [10, 50]]) == 0                  # 4 px is allowed
    assert drop([[10, 10], [96.01, 10], [50, 50], [10, 50]]) == 1                # x > width - 4
    assert drop([[10, 10], [96.0, 10], [50, 50], [10, 50]]) == 0
    assert drop([[10, 10], [50, 10], [50, 76.5], [10, 50]]) == 1                 # y > height - 4
    assert drop([[10, 3.0], [50, 10], [50, 50], [10, 50]], ham=2, tag_id=40) == 1   # the border rule comes first
    assert drop(ok, ham=2, tag_id=40) == 2                                       # then goodness
    assert drop(ok, ham=1, tag_id=36) == 3                                       # then the id limit, on any board size
    assert drop(ok, ham=1, tag_id=35) == 0

    def verdict(ids):
        a = np.asarray(ids, np.int32)
        return lib().ag_frame_verdict(len(a), a.ctypes.data)
    assert verdict([]) == 1 and verdict([0, 1, 2]) == 1
    assert verdict([0, 1, 2, 3]) == 0 and verdict([5, 9, 30, 2, 17]) == 0
    assert verdict([0, 1, 2, 1]) == 2
    assert verdict([4, 4, 4]) == 1                                               # too few is decided before duplicates


def numpy_scene_points(tag_m, nx, ny):
    """InitializeAprilBoard: tag t = nx y + x, corner i at (x s 1.3 + {0, s, s, 0}[i], y s 1.3 + {0, 0, s, s}[i], 0) as cv::Point3f."""
    out = {}
    for y in range(ny):
        for x in range(nx):
            t = nx * y + x
            for i in range(4):
                p = np.float32([x * tag_m * 1.3 + [0, tag_m, tag_m, 0][i], y * tag_m * 1.3 + [0, 0, tag_m, tag_m][i], 0.0])
                out[str((t << 2) + i)] = [float(v) for v in p]
    return out


@pytest.mark.parametrize("tag_m,nx,ny", [(0.04, 6, 6), (0.088, 6, 6), (0.025, 4, 3), (0.03, 7, 8)])
def test_scene_points(tag_m, nx, ny):
    ex = object.__new__(calibrator.AprilGridExtractor)      # scene_points needs no device
    ex.tag_size_m, ex.tags_x, ex.tags_y = tag_m, nx, ny
    pts = ex.scene_points()
    assert pts == numpy_scene_points(tag_m, nx, ny)
    assert sorted(pts, key=int) == [str(i) for i in range(4 * nx * ny)]
    assert pts["1"][0] == float(np.float32(tag_m)) and pts["5"][0] != pts["4"][0]
    np.testing.assert_allclose(np.array([pts[str(i)] for i in range(4 * nx * ny)]), syn.aprilgrid_board_points(nx, ny, tag_m), atol=1e-7)


def test_renderer_draws_opencv_tags(golden):
    # the renderer's tag pattern is the fixture's: the frontal OpenCV frame and a render through the same pinhole agree on
    # the data cells of every tag (sampled at the cell centres)
    from openimucameracalibrator_b200 import camera_models as cm
    shade = lambda x, y: syn.aprilgrid_shade(np.array([x]), np.array([y]), 6, 6, 0.04)[0]  # noqa: E731
    for t in (0, 7, 35):
        c = codes()[t]
        x0, y0 = (t % 6) * 0.052, (t // 6) * 0.052
        for k in range(36):
            r, col = divmod(k, 6)
            x, y = x0 + (2 + col + 0.5) * 0.004, y0 + (7 - r + 0.5) * 0.004
            assert shade(x, y) == ((c >> (35 - k)) & 1)
    assert shade(-0.006, -0.006) == 0.0 and shade(0.0455, 0.0455) == 0.0 and shade(0.0455, 0.02) == 1.0
    assert cm.PINHOLE is not None


def test_capi_rejects_bad_arguments_without_a_device():
    lib_ = calibrator.load_library()
    h = ctypes.c_void_p()
    lib_.icc_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int]
    st = lib_.icc_create(ctypes.byref(h), -1)   # host-only handle
    if st != 0:
        pytest.skip("this build cannot create a host-only handle")
    f = lib_.icc_extract_aprilgrid
    f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                  ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    img = np.zeros((2, 40, 50), np.uint8); uv = np.zeros(2 * 144 * 2); status = np.zeros(2 * 144, np.int32); found = np.zeros(2, np.int32)
    ok = (h, 2, 50, 40, 50, img.ctypes.data, 6, 6, 1.0, uv.ctypes.data, status.ctypes.data, found.ctypes.data, None)
    bad = [dict(i=6, v=0), dict(i=7, v=0), dict(i=6, v=65), dict(i=8, v=0.5), dict(i=8, v=float("nan")), dict(i=8, v=float("inf")),
           dict(i=4, v=49), dict(i=1, v=-1), dict(i=9, v=None), dict(i=10, v=None), dict(i=11, v=None), dict(i=5, v=None)]
    for b in bad:
        args = list(ok); args[b["i"]] = b["v"]
        assert f(*args) == 1, b        # ICC_ERR_INVALID_ARGUMENT
    assert f(*ok) == 2                 # ICC_ERR_NO_DEVICE
    lib_.icc_destroy.argtypes = [ctypes.c_void_p]
    lib_.icc_destroy(h)
