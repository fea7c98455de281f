"""Shared pieces of tests/test_outlier_corners.py: the outlier oracle (tests/outliers/outlier_oracle.cpp), gross corner outliers injected
into a synthetic sequence, the NumPy statement of the rejection rule and the filtered inputs of a rejection."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from openimucameracalibrator_b200 import _capi as capi

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def new_outlier_oracle() -> capi.CApi:
    """the CPU oracle with every camera model, the tangent residual and the rejection entry points, built once per process"""
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="icc_outlier_oracle_"), "libicc_outlier_oracle.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(HERE, "outliers", "outlier_oracle.cpp")])
        _LIB = ctypes.CDLL(out)
    o = capi.CApi(_LIB, "icco_", 0)
    return o


def reject_at(o, threshold_px) -> dict:
    """the oracle's rejection with a given threshold (shards whose sums the caller added up)"""
    s = capi.OutlierSummary()
    o._call("reject_outlier_corners_at", [ctypes.c_double, ctypes.POINTER(capi.OutlierSummary)], float(threshold_px), ctypes.byref(s))
    return s.as_dict()


def inject_outliers(ds, fraction=0.01, lo_px=20.0, hi_px=60.0, seed=5):
    """a copy of `ds` with about `fraction` of the corners displaced by lo_px..hi_px in a random direction, and their indices"""
    rng = np.random.default_rng(seed)
    n = len(ds["point_ids"])
    idx = np.sort(rng.choice(n, size=max(1, int(round(fraction * n))), replace=False))
    ang = rng.uniform(0.0, 2 * np.pi, idx.size); r = rng.uniform(lo_px, hi_px, idx.size)
    out = dict(ds)
    uv = np.array(ds["uv"], dtype=np.float64).reshape(-1, 2).copy()
    uv[idx, 0] += r * np.cos(ang); uv[idx, 1] += r * np.sin(ang)
    out["uv"] = uv
    return out, idx


def numpy_rule(err_pairs, k_sigma, min_px):
    """(kept mask, threshold, rms) of the rejection rule over (n, 2) residual pairs"""
    rx, ry = err_pairs[:, 0], err_pairs[:, 1]
    e = np.sqrt(rx * rx + ry * ry)
    zero = (rx == 0.0) | (ry == 0.0)
    failed = (rx == 1e10) & (ry == 1e10)
    counted = ~zero & ~failed
    rms = float(np.sqrt(np.sum(e[counted] ** 2) / counted.sum())) if counted.any() else 0.0
    thr = max(min_px, k_sigma * rms)
    return zero | (~failed & ~(e > thr)), thr, rms


def filtered(ds, status):
    """the inputs without the corners `status` marks rejected (0); frames keep their place, emptied ones included"""
    keep = status != 0
    off = np.asarray(ds["corner_offsets"])
    counts = np.array([keep[off[i]:off[i + 1]].sum() for i in range(len(off) - 1)])
    out = dict(ds)
    out["corner_offsets"] = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    out["point_ids"] = np.asarray(ds["point_ids"])[keep]
    out["uv"] = np.asarray(ds["uv"], dtype=np.float64).reshape(-1, 2)[keep]
    return out


def copy_state(src, dst):
    """knots, T_i_c, line delay and gravity of one handle / oracle into another"""
    so3, r3, ba, bg = src.get_knots()
    dst.set_knots(so3, r3, ba, bg)
    dst.set_T_i_c(src.get_T_i_c())
    dst.set_line_delay(src.get_line_delay())
    dst.set_known_gravity_dir(src.get_gravity())


def outlier_sequence():
    """the sequence of the sharded tests: 40 views of 6 x 5 corners, 1 % of them gross outliers"""
    from openimucameracalibrator_b200 import camera_models as cm, synthetic as syn
    clean = syn.make_dataset(syn.tiny_config(cm.DIVISION_UNDISTORTION, (437.1, 1.0, 489.1, 270.9, -1.44e-6), n_frames=40, grid=(6, 5)))
    return inject_outliers(clean)[0]


def solve_with_rejection(g):
    """stage 1, one rejection, then 10 LM iterations on the reduced set (a fixed count: where a convergence test stops depends on the last
    digits of the path) -> (summary of the rejection, iterations run, this shard's residual pairs the rejection saw)"""
    F_STAGE1 = capi.FLAG_SPLINE | capi.FLAG_T_I_C
    g.optimize(50, F_STAGE1)
    pairs = g.evaluate(F_STAGE1, gradient=False)[1][:g.num_residuals()[0]].reshape(-1, 2)
    s = g.reject_outlier_corners(3.0, 1.0)
    return s, g.lm_iterations(10, F_STAGE1).iterations, pairs


def shard_worker(rank, world, port, out_dir, mode):
    """One rank of a sharded rejection (mp.spawn).  mode "gloo": both ranks on device 0, the cross-rank sums through the caller hook over
    a gloo group (host copies); "nccl_hook": rank r on device r, the hook over NCCL on the solver stream; "native": the library's NCCL
    communicator.  Writes this rank's corner status, rejection summary, re-solve iterations and T_i_c."""
    import sys
    sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, HERE)
    import torch
    import torch.distributed as dist
    from openimucameracalibrator_b200 import calibrator
    from openimucameracalibrator_b200.distributed import DevicePointer, make_allreduce_hook, make_comm
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dev = 0 if mode == "gloo" else rank
    torch.cuda.set_device(dev)
    if mode == "gloo":
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    lib = calibrator.load_library()
    ds = outlier_sequence()
    g = capi.CApi(lib, "icc_", dev)
    if mode == "native":
        capi.load_dataset(g, ds, comm=make_comm(lib, dev))
    else:
        capi.load_dataset(g, ds, shard=(rank, world))
        if mode == "nccl_hook":
            g.set_allreduce(make_allreduce_hook(g.get_stream(), dev))
        else:
            ext = torch.cuda.ExternalStream(g.get_stream(), device=f"cuda:{dev}")

            def hook(ptr, n, stream, user):   # the sum on the host: the solver stream drained, summed, copied back before the call returns
                t = torch.as_tensor(DevicePointer(ptr, n), device=f"cuda:{dev}")
                ext.synchronize()
                h = t.cpu()
                dist.all_reduce(h)
                t.copy_(h)
                torch.cuda.synchronize(dev)
            g.set_allreduce(hook)
    s, iters, pairs = solve_with_rejection(g)
    np.save(os.path.join(out_dir, f"pairs{rank}.npy"), pairs)
    np.save(os.path.join(out_dir, f"status{rank}.npy"), g.corner_status())
    np.save(os.path.join(out_dir, f"summary{rank}.npy"), np.array([s["n_corners"], s["n_rejected"], s["n_failed"], s["n_frames_emptied"], s["rms_px"],
                                                                    s["threshold_px"], iters] + list(g.get_T_i_c())))
    g.close()
    dist.destroy_process_group()
