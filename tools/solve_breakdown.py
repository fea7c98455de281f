#!/usr/bin/env python
"""Where the time of the damped linear solve goes inside an LM step, per kernel, on the GPU.

Loads a BASELINE config (default 4), runs warm-up LM iterations, then records K more under torch.profiler with CUDA activities and
writes the Chrome trace to OUT/solve_breakdown_trace.json (OUT defaults to a directory under the system's temporary directory).
For every solve (prepare_kernel ... finish_kernel) it prints per kernel the median duration and the median distance from its
predecessor's end to its own end (the reduction and back-substitution levels listed one by one), then the spans: the whole solve,
the forward part (prepare start -> root end), the backward sweep (first back-substitution kernel start -> finish_kernel end) and
the part of that sweep left once the root is solved (root end -> finish end).  Under programmatic dependent launch a kernel starts
while its predecessor still runs and waits inside, so durations include that wait and their sums exceed the spans; the distances
between consecutive ends are the critical path.

    python tools/solve_breakdown.py [--config 4] [--iters 6] [--warmup 2] [--out DIR]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SOLVER_KERNELS = ("prepare_kernel", "eliminate_kernel", "reduce_kernel", "root_kernel", "backsub", "finish_kernel")


def short_name(full):
    """`void icc::(anonymous namespace)::backsub_kernel<false>(...)` -> `backsub_kernel<false>`"""
    s = full.replace("(anonymous namespace)", "")
    s = s[5:] if s.startswith("void ") else s
    return s.split("(")[0].split("::")[-1]


def gpu_identity():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001 -- the identity line is informational
        return f"nvidia-smi unavailable: {e}"


def split_solves(kernels):
    """kernels: [(name, start_us, dur_us)] sorted by start -> one list per solve, prepare_kernel .. finish_kernel inclusive."""
    solves, cur = [], None
    for k in kernels:
        if k[0].startswith("prepare_kernel"):
            cur = [k]
        elif cur is not None:
            cur.append(k)
            if k[0].startswith("finish_kernel"):
                solves.append(cur); cur = None
    return solves


def label(solve):
    """Stable per-solve labels: repeated kernels get their launch index (reduce_kernel#1 = level 1, backsub_kernel<false>#1 = level L)."""
    seen, out = {}, []
    for name, t, d in solve:
        i = seen.get(name, 0) + 1; seen[name] = i
        out.append((f"{name}#{i}" if name.startswith(("reduce_kernel", "backsub")) else name, t, d))
    return out


def median(v):
    v = sorted(v); n = len(v)
    return 0.5 * (v[(n - 1) // 2] + v[n // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=4)
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "solve_breakdown"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from openimucameracalibrator_b200 import _capi as capi, calibrator, synthetic as syn

    if not torch.cuda.is_available():
        raise SystemExit("solve_breakdown.py needs a CUDA device")
    flags = capi.FLAG_SPLINE | capi.FLAG_T_I_C
    ds = syn.make_dataset(syn.CONFIGS[args.config])
    api = capi.CApi(calibrator.load_library(), "icc_", 0)
    capi.load_dataset(api, ds)
    so3, r3, ba, bg = api.get_knots(); T0 = api.get_T_i_c(); ld0 = api.get_line_delay()

    def reset():
        api.set_knots(so3, r3, ba, bg); api.set_T_i_c(T0); api.set_line_delay(ld0)

    for _ in range(args.warmup):
        reset(); api.lm_iterations(1, flags)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            reset(); api.lm_iterations(1, flags)
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "solve_breakdown_trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f)["traceEvents"]
    kernels = sorted(((short_name(e["name"]), float(e["ts"]), float(e["dur"])) for e in events
                      if e.get("cat") == "kernel" and any(s in e["name"] for s in SOLVER_KERNELS)), key=lambda k: k[1])
    solves = [label(s) for s in split_solves(kernels)]
    if not solves:
        raise SystemExit("no complete solve (prepare_kernel .. finish_kernel) in the trace")

    per_kernel, order = {}, []
    spans = {"solve": [], "forward": [], "backward_sweep": [], "after_root": []}
    for s in solves:
        for name, t, d in s:
            if name not in per_kernel:
                per_kernel[name] = []; order.append(name)
            per_kernel[name].append(d)
        end = lambda k: k[1] + k[2]   # noqa: E731
        root = next(k for k in s if k[0] == "root_kernel")
        first_back = next((k for k in s if k[0].startswith("backsub")), s[-1])
        spans["solve"].append(end(s[-1]) - s[0][1])
        spans["forward"].append(end(root) - s[0][1])
        spans["backward_sweep"].append(end(s[-1]) - first_back[1])
        spans["after_root"].append(end(s[-1]) - end(root))

    print(f"gpu: {gpu_identity()}")
    print(f"config {args.config}: {len(solves)} solves profiled (medians over solves, microseconds)")
    print(f"{'kernel':32s} {'median':>9s} {'min':>9s} {'max':>9s} {'end-to-end':>10s}")
    for name in order:
        v = per_kernel[name]
        step = [x[1] + x[2] - (y[1] + y[2]) for s in solves for x, y in zip(s[1:], s) if x[0] == name]   # end minus predecessor's end
        print(f"{name:32s} {median(v):9.2f} {min(v):9.2f} {max(v):9.2f} {median(step) if step else 0.0:10.2f}")
    busy = {"forward": 0.0, "backward_sweep": 0.0}
    for name in order:
        busy["backward_sweep" if re.match(r"(backsub|finish)", name) else "forward"] += median(per_kernel[name])
    for k, v in spans.items():
        extra = f"   (sum of kernel medians {busy[k]:.2f})" if k in busy else ""
        print(f"span {k:27s} {median(v):9.2f} {min(v):9.2f} {max(v):9.2f}{extra}")
    result = {"config": args.config, "solves": len(solves), "gpu": gpu_identity(),
              "kernels_us": {n: median(per_kernel[n]) for n in order}, "spans_us": {k: median(v) for k, v in spans.items()}}
    with open(os.path.join(args.out, "solve_breakdown.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["spans_us"]))
    print(f"trace: {trace}")


if __name__ == "__main__":
    main()
