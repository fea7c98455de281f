"""The host side of the drop-in extract_board_to_json without a GPU: the PNG decoder (csrc/icc_png.hpp) against committed cv2.imread
output and on malformed files, the colour stage (resize, then BGR2GRAY; icc_board_math.cuh) against committed cv2 output, the UBJSON
writer against io_formats.ubjson_dumps, the corner-file reader on array-form scene_pts, and the CLI's refusals, which all come before
any GPU work."""
import ctypes
import json
import os
import struct
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

import png_support as ps
from openimucameracalibrator_b200 import io_formats

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLI = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "extract_board_to_json")
_LIBS = {}


def cli_lib():
    if "cli" not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_cli_host_"), "libcli_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "board", "cli_host.cpp"), "-lz"])
        lib = ctypes.CDLL(out)
        lib.png_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t] + [ctypes.POINTER(ctypes.c_int)] * 3
        lib.png_result.argtypes = [ctypes.c_void_p]
        lib.last_error.restype = ctypes.c_char_p
        lib.ubjson_from_text.argtypes = [ctypes.c_char_p]
        lib.ubjson_from_text.restype = ctypes.c_longlong
        lib.bytes_result.argtypes = [ctypes.c_void_p]
        lib.scene_points.argtypes = [ctypes.c_char_p, ctypes.c_size_t]
        lib.board_result.argtypes = [ctypes.c_void_p]
        _LIBS["cli"] = lib
    return _LIBS["cli"]


def bgr_lib():
    if "bgr" not in _LIBS:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_bgr_host_"), "libbgr_host.so")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                               "-o", out, os.path.join(HERE, "board", "board_bgr_host.cu")])
        lib = ctypes.CDLL(out)
        lib.bm_bgr_resize_gray.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_void_p]
        _LIBS["bgr"] = lib
    return _LIBS["bgr"]


def decode(data: bytes):
    """-> (image: (h, w) gray or (h, w, 3) BGR, None) or (None, error message)."""
    w, h, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    if not cli_lib().png_decode(data, len(data), ctypes.byref(w), ctypes.byref(h), ctypes.byref(c)):
        return None, cli_lib().last_error().decode()
    out = np.zeros((h.value, w.value, c.value), np.uint8)
    cli_lib().png_result(out.ctypes.data)
    return (out[:, :, 0] if c.value == 1 else out), None


@pytest.fixture(scope="module")
def variants():
    return np.load(os.path.join(HERE, "golden", "png_variants.npz"))


def test_png_variants_decode_like_cv2_imread(variants):
    names = variants["names"]
    assert len(names) > 60
    for k, name in enumerate(names):
        img, err = decode(variants[f"png_{k}"].tobytes())
        assert err is None, (name, err)
        ref = variants[f"img_{k}"]
        gray_type = name.startswith(("t0_", "t4_", "gray"))
        assert img.ndim == (2 if gray_type else 3), name          # gray comes back as one channel, imread replicates it
        full = np.repeat(img[:, :, None], 3, 2) if img.ndim == 2 else img
        np.testing.assert_array_equal(full, ref, err_msg=str(name))


def _valid_png():
    return ps.encode_png(np.arange(5 * 7 * 3).reshape(5, 7, 3) % 256, 2, 8, 4)


def _with_chunk(data: bytes, kind: bytes, body: bytes, before=b"IDAT") -> bytes:
    i = data.index(before) - 4
    return data[:i] + ps.chunk(kind, body) + data[i:]


def _patch_ihdr(width, height):
    d = bytearray(_valid_png())
    body = struct.pack(">IIBBBBB", width, height, 8, 2, 0, 0, 0)
    d[16:29] = body
    d[29:33] = struct.pack(">I", zlib.crc32(b"IHDR" + body) & 0xFFFFFFFF)
    return bytes(d)


def _malformed():
    good = _valid_png()
    idat = good.index(b"IDAT") - 4
    n = struct.unpack(">I", good[idat:idat + 4])[0]
    z = good[idat + 8:idat + 8 + n]
    excess = good[:idat] + ps.chunk(b"IDAT", z + b"\x00\x01") + good[idat + 12 + n:]
    raw = zlib.decompress(z)
    longer = good[:idat] + ps.chunk(b"IDAT", zlib.compress(raw + b"\x00" * 22)) + good[idat + 12 + n:]
    shorter = good[:idat] + ps.chunk(b"IDAT", zlib.compress(raw[:-5])) + good[idat + 12 + n:]
    exif6 = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, 6, 0) + struct.pack("<I", 0)
    flipped = bytearray(good); flipped[idat + 10] ^= 0x40
    return [
        ("bad signature", b"\x89PNX" + good[4:], "signature"),
        ("crc flip", bytes(flipped), "CRC"),
        ("truncated in IDAT", good[:idat + 20], "truncated"),
        ("truncated before IEND", good[:-12], "IEND"),
        ("truncated stream", good[:idat] + ps.chunk(b"IDAT", z[:len(z) // 2]) + good[idat + 12 + n:], "truncated"),
        ("excess after the stream", excess, "excess"),
        ("excess image data", longer, "excess"),
        ("too little image data", shorter, "truncated"),
        ("zero width", _patch_ihdr(0, 5), "zero"),
        ("zero height", _patch_ihdr(7, 0), "zero"),
        ("absurd size", _patch_ihdr(1 << 30, 1 << 30), "too large"),
        ("unknown critical chunk", _with_chunk(good, b"QUUX", b"abc"), "critical"),
        ("exif orientation 6", _with_chunk(good, b"eXIf", exif6), "orientation"),
        ("empty", b"", "signature"),
    ]


@pytest.mark.parametrize("name,data,word", _malformed(), ids=[m[0] for m in _malformed()])
def test_malformed_png_is_an_error_naming_the_file(name, data, word):
    img, err = decode(data)
    assert img is None and err.startswith("test.png: ") and word in err, (name, err)


def test_unknown_ancillary_chunk_is_skipped():
    good = _valid_png()
    img, err = decode(_with_chunk(good, b"quUx", b"whatever"))
    ref, _ = decode(good)
    assert err is None
    np.testing.assert_array_equal(img, ref)


def test_bgr_resize_then_gray_equals_committed_cv2():
    g = np.load(os.path.join(HERE, "golden", "bgr_resize_gray_opencv.npz"))
    bgr = g["bgr"]
    for f in g["factors"]:
        ref = g["gray_" + f"{f:g}".replace(".", "p")]
        for k in range(len(bgr)):
            img = np.ascontiguousarray(bgr[k])
            h, w = img.shape[:2]
            out = np.zeros(ref.shape[1:], np.uint8)
            bgr_lib().bm_bgr_resize_gray(img.ctypes.data, 3 * w, w, h, float(f), out.ctypes.data)
            np.testing.assert_array_equal(out, ref[k], err_msg=f"f = {f}")
    # gray replicated to B = G = R converts to itself, so a gray PNG may take the gray entry
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    out = np.zeros_like(v)
    rep = np.ascontiguousarray(np.repeat(v[:, :, None], 3, 2))
    bgr_lib().bm_bgr_resize_gray(rep.ctypes.data, 48, 16, 16, 1.0, out.ctypes.data)
    np.testing.assert_array_equal(out, v)


def _ubjson(doc):
    lib = cli_lib()
    n = lib.ubjson_from_text(json.dumps(doc).encode())
    assert n >= 0, lib.last_error()
    out = np.zeros(n, np.uint8)
    lib.bytes_result(out.ctypes.data)
    return out.tobytes()


def test_ubjson_writer_equals_io_formats():
    s = np.float32(0.0121)
    doc = {"calibration_board_type": 1, "square_size_meter": float(s), "image_width": 640, "image_height": 360, "camera_fps": 29.97,
           "scene_pts": [[float(np.float32(i) * s), float(np.float32(j) * s), 0.0] for i in range(3) for j in range(4)],
           "views": {"1500000.000000": {"image_points": {str(c): [100.25 + c, 7.0 / 3.0] for c in range(12)}}},
           "ints": [0, -1, 127, 128, 255, 256, -128, -129, 32767, 32768, -32769, 2 ** 31 - 1, 2 ** 31, -2 ** 31 - 1, 2 ** 40], "s": "x" * 300,
           "flags": [True, False, None], "empty": {}, "nested": [[], [1.5e-300, -0.0]]}
    assert _ubjson(doc) == io_formats.ubjson_dumps(doc)


def _scene_board(scene):
    lib = cli_lib()
    data = io_formats.ubjson_dumps(scene)
    n = lib.scene_points(data, len(data))
    assert n >= 0, lib.last_error()
    out = np.zeros((n, 4))
    lib.board_result(out.ctypes.data)
    return out


def test_scene_reader_takes_array_and_object_form():
    pts = [[0.1 * i, 0.2 * i, 0.0] for i in range(14 * 9)]
    a = _scene_board({"scene_pts": pts})
    o = _scene_board({"scene_pts": {str(i): p for i, p in enumerate(pts)}})
    np.testing.assert_array_equal(a, o)
    assert a.shape == (126, 4) and (a[:, 3] == 1).all() and np.allclose(a[5, :3], [0.5, 1.0, 0.0])


# ---- the CLI's refusals: none of them needs a GPU -----------------------------------------------------------------------------
def _run(*args):
    return subprocess.run([CLI, *args], capture_output=True, text=True)


def _folder(tmp_path, names):
    d = tmp_path / "frames"
    d.mkdir()
    png = _valid_png()
    for n in names:
        (d / n).write_bytes(png)
    return d


def test_existing_output_is_skipped_untouched(tmp_path):
    out = tmp_path / "corners.uson"
    out.write_bytes(b"previous")
    r = _run("--input_path", str(tmp_path / "missing"), "--board_type", "charuco", "--save_corners_json_path", str(out))
    assert r.returncode == 0 and "Skipping corner extraction. Already extracted for: " in r.stdout, r
    assert out.read_bytes() == b"previous"


@pytest.mark.parametrize("case", ["charuco", "apriltag", "unknown", "default_board_type", "file_path", "missing_folder", "empty_folder", "non_numeric",
                                  "two_timestamps", "factor_below_1", "recompute_with_bad_type"])
def test_refusals_write_nothing(tmp_path, case):
    out = tmp_path / "corners.uson"
    folder = _folder(tmp_path, ["1000000000.png", "1033333333.png", "1066666666.png"])
    args = ["--input_path", str(folder), "--board_type", "radon", "--save_corners_json_path", str(out)]
    word = None
    if case in ("charuco", "apriltag", "unknown"):
        args[3] = case; word = "only the radon"
    elif case == "default_board_type":
        args = args[:2] + args[4:]; word = "only the radon"
    elif case == "file_path":
        args[1] = str(folder / "1000000000.png"); word = "video input is not supported"
    elif case == "missing_folder":
        args[1] = str(tmp_path / "nope"); word = "does not exist"
    elif case == "empty_folder":
        (tmp_path / "empty").mkdir(); args[1] = str(tmp_path / "empty"); word = "No image files found"
    elif case == "non_numeric":
        (folder / "frame_a.png").write_bytes(b""); word = "frame_a.png"
    elif case == "two_timestamps":
        os.remove(folder / "1066666666.png"); (folder / "1033333333.PNG").write_bytes(b""); word = "3 distinct timestamps"
    elif case == "factor_below_1":
        args += ["--downsample_factor", "0.5"]; word = "downsample_factor"
    elif case == "recompute_with_bad_type":
        out.write_bytes(b"previous"); args[3] = "charuco"; args.append("--recompute_corners"); word = "only the radon"
    r = _run(*args)
    assert r.returncode != 0 and word in r.stderr, (case, r)
    if case == "recompute_with_bad_type":
        assert out.read_bytes() == b"previous"
    else:
        assert not out.exists()


def test_aruco_flags_are_accepted():
    r = _run("--aruco_detector_params", "params.yml", "--aruco_dict=3", "--board_type=radon", "--input_path=/nonexistent/frames",
             "--save_corners_json_path=/nonexistent/out.uson", "--verbose", "--num_squares_x=14", "--num_squares_y", "9")
    assert r.returncode != 0 and "does not exist" in r.stderr, r
    assert "unknown command line flag" not in r.stderr
