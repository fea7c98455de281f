"""Writes the fixtures of the drop-in extract_board_to_json:

  png_variants.npz          small PNG files written by tests/png_support.py (every colour type and bit depth, each row filter, Adam7,
                            IDAT in several chunks, PLTE with and without tRNS, gray and RGB with tRNS, odd sizes), each with what
                            cv2.imread(path, IMREAD_COLOR) returns for it;
  bgr_resize_gray_opencv.npz colour-tinted radon renders at 640 x 480, with cvtColor(resize(bgr, 1/f), BGR2GRAY) at f in 1, 1.5, 2, 2.5, 3, 4,
                            the order BoardExtractor::ExtractImageFolderToJson runs them in.

Run once where cv2 is importable (python tests/golden/make_png_golden.py); no test imports cv2.
"""
import os
import struct
import sys
import tempfile

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import png_support as ps  # noqa: E402
from openimucameracalibrator_b200 import camera_models as cm, synthetic as syn  # noqa: E402

FACTORS = (1.0, 1.5, 2.0, 2.5, 3.0, 4.0)
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}


def exif(orientation):
    return b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack("<I", 0)


def variants():
    rng = np.random.default_rng(7)
    out = []

    def samples(ctype, depth, h, w):
        c = ps.CHANNELS[ctype]
        hi = (1 << depth) if ctype != 3 else 1 << min(depth, 8)
        s = rng.integers(0, hi, (h, w, c))
        return s[:, :, 0] if c == 1 else s

    def palette(n):
        return rng.integers(0, 256, (n, 3))

    for ctype, depths in DEPTHS.items():
        for depth in depths:
            for (h, w) in ((13, 11), (6, 37)):
                s = samples(ctype, depth, h, w)
                pal = palette(1 << depth) if ctype == 3 else None
                rows = lambda p, y: y % 5  # noqa: E731   every filter type, row by row
                out.append((f"t{ctype}_d{depth}_{h}x{w}_rowfilters", ps.encode_png(s, ctype, depth, rows, palette=pal)))
                out.append((f"t{ctype}_d{depth}_{h}x{w}_adam7", ps.encode_png(s, ctype, depth, rows, interlace=True, palette=pal)))
    s = samples(2, 8, 17, 23)
    for f in range(5):
        out.append((f"rgb8_filter{f}", ps.encode_png(s, 2, 8, f)))
    out.append(("rgb8_idat7", ps.encode_png(s, 2, 8, 4, idat_chunks=7, level=9)))
    out.append(("rgb8_adam7_idat3", ps.encode_png(s, 2, 8, 1, interlace=True, idat_chunks=3)))
    for (h, w) in ((1, 1), (2, 3), (5, 1), (1, 9)):   # Adam7 with empty passes
        out.append((f"rgb8_adam7_{h}x{w}", ps.encode_png(samples(2, 8, h, w), 2, 8, 4, interlace=True)))
        out.append((f"gray1_adam7_{h}x{w}", ps.encode_png(samples(0, 1, h, w), 0, 1, 3, interlace=True)))
    idx = rng.integers(0, 16, (9, 14))
    out.append(("palette4_trns", ps.encode_png(idx, 3, 4, 2, palette=palette(16), trns=bytes(rng.integers(0, 256, 10, dtype=np.uint8)))))
    out.append(("palette8_short_palette", ps.encode_png(rng.integers(0, 40, (9, 14)), 3, 8, 0, palette=palette(40))))
    out.append(("gray8_trns", ps.encode_png(samples(0, 8, 9, 14), 0, 8, 4, trns=struct.pack(">H", 77))))
    out.append(("gray2_trns", ps.encode_png(samples(0, 2, 9, 14), 0, 2, 4, trns=struct.pack(">H", 1))))
    out.append(("gray16_trns", ps.encode_png(samples(0, 16, 9, 14), 0, 16, 4, trns=struct.pack(">H", 4000))))
    out.append(("rgb8_trns", ps.encode_png(samples(2, 8, 9, 14), 2, 8, 4, trns=struct.pack(">HHH", 1, 2, 3))))
    out.append(("rgb8_exif_orientation1_text", ps.encode_png(samples(2, 8, 9, 14), 2, 8, 4, extra_chunks=[(b"eXIf", exif(1)), (b"tEXt", b"Comment\x00x")],
                                                              after_idat=[(b"tIME", struct.pack(">HBBBBB", 2024, 5, 17, 12, 30, 0))])))
    return out


def bgr_renders():
    frames = []
    size = (640, 480)
    cams = [(cm.PINHOLE, (560.0, 1.0, 0.0, 322.0, 238.0, -0.05, 0.01)), (cm.FISHEYE, (290.0, 1.0, 0.0, 318.0, 242.0, 0.05, 0.07, -0.11, 0.05))]
    tints = [((0.55, 25.0), (0.95, 5.0), (0.75, 40.0)), ((1.0, 0.0), (0.6, 60.0), (0.35, 10.0))]   # (gain, offset) per B, G, R
    for (model, intr), tint, (dist, tilt, axis, roll) in zip(cams, tints, ((0.9, 25.0, 30.0, 10.0), (0.45, 35.0, 120.0, 200.0))):
        R, t = syn.radon_view_pose(14, 9, 0.03, dist, tilt, axis, roll)
        g, _, _ = syn.render_radon_board(model, intr, size, R, t, 14, 9, 0.03, supersample=2, blur_sigma_px=0.6)
        ramp = np.linspace(-20, 20, size[0])[None, :]
        ch = [np.clip(gain * g + off + k * ramp, 0, 255) for k, (gain, off) in zip((1, 0, -1), tint)]
        frames.append(np.rint(np.stack(ch, -1)).astype(np.uint8))
    return np.stack(frames)


def main():
    tmp = tempfile.mkdtemp()
    names, files, imgs = [], {}, {}
    for k, (name, data) in enumerate(variants()):
        path = os.path.join(tmp, f"{k}.png")
        with open(path, "wb") as f:
            f.write(data)
        img = cv2.imread(path, cv2.IMREAD_COLOR)
        assert img is not None, name
        names.append(name)
        files[f"png_{k}"] = np.frombuffer(data, np.uint8)
        imgs[f"img_{k}"] = img
    np.savez_compressed(os.path.join(HERE, "png_variants.npz"), names=np.array(names), opencv_version=cv2.__version__, **files, **imgs)
    bgr = bgr_renders()
    gray = {}
    for f in FACTORS:
        key = f"gray_{f:g}".replace(".", "p")
        gray[key] = np.stack([cv2.cvtColor(cv2.resize(b, None, fx=1.0 / f, fy=1.0 / f), cv2.COLOR_BGR2GRAY) if f != 1.0 else cv2.cvtColor(b, cv2.COLOR_BGR2GRAY)
                              for b in bgr])
    np.savez_compressed(os.path.join(HERE, "bgr_resize_gray_opencv.npz"), bgr=bgr, factors=np.array(FACTORS), opencv_version=cv2.__version__, **gray)
    print(len(names), "PNG variants;", bgr.shape, "BGR frames")


if __name__ == "__main__":
    main()
