"""Wall time of the drop-in extract_board_to_json on a folder of 1920 x 1080 colour PNG frames, and where it goes.

Writes N frames (default 600) as <timestamp_ns>.png with tests/png_support.py at zlib level 1 (cv::imwrite's default) and Paeth rows:
eight tinted radon renders, each frame one of them with its own 1 DN noise, so that every file is different and compresses like a camera
frame.  Then runs `bin/extract_board_to_json --board_type radon --downsample_factor 2` and reports, as one JSON line:
  wall seconds and frames/s, decode seconds summed over the threads and per thread, GPU seconds (the extraction calls), the thread and
  host core counts, and the GPU's name, power limit and clocks (nvidia-smi, read in the same run).
With --reference and cv2 importable it also times the reference's per-frame work on the first --reference_frames files:
cv2.imread + cv2.resize + cvtColor(BGR2GRAY) + findChessboardCornersSB(CALIB_CB_LARGER | CALIB_CB_MARKER | CALIB_CB_EXHAUSTIVE).

    python tools/extract_board_folder_timing.py [--frames 600] [--out board_folder_timing.json]
"""
import argparse
import json
import multiprocessing as mp
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import png_support as ps  # noqa: E402
from openimucameracalibrator_b200 import camera_models as cm, synthetic as syn  # noqa: E402

SIZE = (1920, 1080)
W, H, SQ = 14, 9, 0.0121
_BASE = None


def _renders():
    intr = (1350.0, 1.0, 0.0, 960.0, 540.0, 0.0, 0.0)
    rng = np.random.default_rng(0)
    out = []
    for k in range(8):
        R, t = syn.radon_view_pose(W, H, SQ, rng.uniform(0.25, 0.32), rng.uniform(5, 35), rng.uniform(0, 360), rng.uniform(-20, 20))
        g, _, _ = syn.render_radon_board(cm.PINHOLE, intr, SIZE, R, t, W, H, SQ, supersample=1, blur_sigma_px=0.8)
        out.append(np.stack([np.clip(a * g + b, 0, 255) for a, b in ((0.6, 30.0), (0.9, 10.0), (0.7, 45.0))], -1).astype(np.float32))
    return out


def _init(base):
    global _BASE
    _BASE = base


def _write(args):
    k, path = args
    rng = np.random.default_rng(k)
    img = np.clip(_BASE[k % len(_BASE)] + rng.normal(0.0, 1.0, _BASE[0].shape).astype(np.float32), 0, 255)
    ps.write_png(path, np.rint(img).astype(np.uint8), level=1, filters=4)


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--factor", type=float, default=2.0)
    ap.add_argument("--reference", action="store_true", help="also time the reference's per-frame OpenCV work (needs cv2)")
    ap.add_argument("--reference_frames", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="icc_board_folder_")
    frames = os.path.join(tmp, "frames")
    os.makedirs(frames)
    t0 = time.time()
    base = _renders()
    paths = [os.path.join(frames, f"{1_700_000_000_000_000_000 + k * 33_333_333}.png") for k in range(a.frames)]
    with mp.Pool(os.cpu_count(), initializer=_init, initargs=(base,)) as pool:
        pool.map(_write, list(enumerate(paths)), chunksize=4)
    write_s = time.time() - t0
    mb = sum(os.path.getsize(p) for p in paths) / 1e6
    out = os.path.join(tmp, "corners.uson")
    cli = os.path.join(ROOT, "openimucameracalibrator_b200", "bin", "extract_board_to_json")
    t0 = time.time()
    r = subprocess.run([cli, "--input_path", frames, "--board_type", "radon", "--num_squares_x", str(W), "--num_squares_y", str(H),
                        "--checker_square_length_m", str(SQ), "--downsample_factor", str(a.factor), "--save_corners_json_path", out], capture_output=True, text=True)
    wall = time.time() - t0
    if r.returncode != 0:
        sys.exit(r.stderr + r.stdout)
    m = re.search(r"Found the board in (\d+) of (\d+) frames; wall ([\d.e+-]+) s, decode ([\d.e+-]+) s summed over (\d+) threads, GPU ([\d.e+-]+) s", r.stdout)
    found, n, cli_wall, decode_s, threads, gpu_s = int(m[1]), int(m[2]), float(m[3]), float(m[4]), int(m[5]), float(m[6])
    res = dict(frames=n, found=found, size=list(SIZE), factor=a.factor, png_mb=round(mb, 1), write_seconds=round(write_s, 1),
               process_wall_s=round(wall, 3), cli_wall_s=round(cli_wall, 3), frames_per_s=round(n / cli_wall, 1), decode_s_total=round(decode_s, 3),
               threads=threads, decode_s_per_thread=round(decode_s / threads, 3), decode_ms_per_frame_one_thread=round(1e3 * decode_s / n, 2),
               gpu_s=round(gpu_s, 3), gpu_fraction_of_wall=round(gpu_s / cli_wall, 3), host_cores=os.cpu_count(), gpu=_gpu_info())
    if a.reference:
        try:
            import cv2
            flags = cv2.CALIB_CB_LARGER | cv2.CALIB_CB_MARKER | cv2.CALIB_CB_EXHAUSTIVE
            t0 = time.time()
            for p in paths[:a.reference_frames]:
                img = cv2.resize(cv2.imread(p), None, fx=1.0 / a.factor, fy=1.0 / a.factor)
                cv2.findChessboardCornersSBWithMeta(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), (W, H), flags)
            res["reference_s_per_frame"] = round((time.time() - t0) / a.reference_frames, 3)
            res["opencv_threads"] = cv2.getNumThreads()
        except ImportError:
            res["reference_s_per_frame"] = "cv2 not importable"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
