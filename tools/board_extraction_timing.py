"""Device throughput of icc_extract_radon_board at 960x540: 3000 frames (eight rendered radon-board views, repeated) as one torch
CUDA tensor, timed with a host clock around calls that end in a device synchronise; and, when cv2 is importable,
cv2.findChessboardCornersSB with the reference's flags on the same eight frames on this host's cores.

    python tools/board_extraction_timing.py [--frames 3000] [--rounds 3] [--out board_timing.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from openimucameracalibrator_b200 import calibrator, camera_models as cm, synthetic as syn  # noqa: E402
from openimucameracalibrator_b200._capi import CApi  # noqa: E402

W, H, SQ = 14, 9, 0.03
CAM = (cm.FISHEYE, (435.5, 1.0, 0.0, 479.1, 274.5, 0.05, 0.07, -0.11, 0.05))


def frames8():
    out = []
    for k in range(8):
        R, t = syn.radon_view_pose(W, H, SQ, 0.45 + 0.03 * k, 10.0 + 5 * k, 45.0 * k, 30.0 * k)
        out.append(syn.render_radon_board(CAM[0], CAM[1], (960, 540), R, t, W, H, SQ, supersample=2, blur_sigma_px=0.6, noise_sigma_dn=1.0, seed=k)[0])
    return np.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    base = frames8()
    reps = (a.frames + 7) // 8
    dev = torch.from_numpy(base).cuda().repeat(reps, 1, 1)[:a.frames].contiguous()
    api = CApi(calibrator.load_library(), "icc_", 0)
    uv, found, s = api.extract_radon_board(dev[:64], W, H)   # warm-up: module load, allocator
    times = []
    for _ in range(a.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        uv, found, s = api.extract_radon_board(dev, W, H)
        times.append(time.perf_counter() - t0)
    res = dict(gpu=gpu, frames=a.frames, size=[960, 540], seconds=times, fps_median=a.frames / float(np.median(times)), found=int(found.sum()),
               summary=s)
    try:
        import cv2
        flags = cv2.CALIB_CB_LARGER | cv2.CALIB_CB_MARKER | cv2.CALIB_CB_EXHAUSTIVE
        t0 = time.perf_counter()
        ok = [cv2.findChessboardCornersSB(f, (W, H), flags)[0] for f in base]
        dt = (time.perf_counter() - t0) / len(base)
        res["opencv"] = dict(seconds_per_frame=dt, found=int(sum(ok)), threads=cv2.getNumThreads(), cores=os.cpu_count())
    except ImportError:
        res["opencv"] = "not measured: cv2 is not importable here"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
