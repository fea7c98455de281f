"""Throughput of icc_extract_aprilgrid on one GPU: frames/s for AprilGrid renders already on the device, at 960 x 540 and
1920 x 1080, with the card's name and power limit.

    python tools/aprilgrid_timing.py [--frames 512] [--repeats 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openimucameracalibrator_b200 import calibrator, camera_models as cm, synthetic as syn  # noqa: E402
from openimucameracalibrator_b200._capi import CApi  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def views(size, n_distinct=8):
    w, h = size
    f = 820.0 * w / 960.0
    intr = (f, 1.0, 0.0, w / 2.0, h / 2.0, -0.05, 0.01)
    rays = syn.camera_rays(cm.PINHOLE, intr, size, 2)
    rng = np.random.default_rng(1)
    out = []
    for k in range(n_distinct):
        R, t = syn.aprilgrid_view_pose(6, 6, 0.04, rng.uniform(0.45, 0.7), rng.uniform(0, 35), rng.uniform(0, 360), rng.uniform(-40, 40))
        out.append(syn.render_aprilgrid(cm.PINHOLE, intr, size, R, t, supersample=2, blur_sigma_px=0.6, noise_sigma_dn=2.0, seed=k, rays=rays)[0])
    return np.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    api = CApi(calibrator.load_library(), "icc_", 0)
    res = {"card": card(), "frames": a.frames, "sizes": {}}
    for size in ((960, 540), (1920, 1080)):
        base = views(size)
        frames = torch.from_numpy(np.concatenate([base] * (a.frames // len(base)))).cuda()
        api.extract_aprilgrid(frames[:16], 6, 6)           # warm-up: allocations and module load
        best, found = 1e30, 0
        for _ in range(a.repeats):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, _, fd, s = api.extract_aprilgrid(frames, 6, 6)
            best = min(best, time.perf_counter() - t0)
            found = int(fd.sum())
        res["sizes"][f"{size[0]}x{size[1]}"] = {"seconds": best, "frames_per_s": frames.shape[0] / best, "found": found,
                                                "n_frames": int(frames.shape[0]), "gpu_launches": s["gpu_launches"]}
        print(f"{size[0]}x{size[1]}: {frames.shape[0]} frames in {best:.3f} s = {frames.shape[0] / best:.0f} frames/s, {found} found")
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
