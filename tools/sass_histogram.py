#!/usr/bin/env python
"""Per-kernel SASS opcode histogram of the device objects of libicc_b200.so (cuobjdump -sass): makes the claims of DESIGN.md checkable
from the repository -- FP64 tensor-core MMAs (DMMA, and per shape) in the evaluation / solver kernels, shared-memory parking (LDS / STS) in
eval_tmem_kernel, no local-memory spills (LDL / STL), no library kernels, no HMMA.
usage: python tools/sass_histogram.py"""
import collections, glob, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = ["DMMA", "DMMA.8x8x4", "DMMA.16x8x4", "DMMA.16x8x8", "DMMA.16x8x16", "DFMA", "DMUL", "DADD", "LDTM", "STTM", "UTCATOMSWS", "REDG", "RED", "ATOMG", "LDS", "STS", "LDG", "STG", "LDL", "STL", "SHFL", "BAR", "MUFU", "HMMA", "UTCHMMA", "UTCQMMA", "UTMALDG", "UBLKCP"]
for obj in sorted(glob.glob(os.path.join(ROOT, "openimucameracalibrator_b200", "csrc", "*.o"))):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    if "Function :" not in out:
        continue
    print(f"== {os.path.basename(obj)}")
    fn, hist = None, {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            fn = re.sub(r"\(icc::.*|\(double.*|\(int.*|\(\)$", "", name.replace("(anonymous namespace)::", "").replace("void ", "").replace("icc::", "", 1))
            hist[fn] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)(\.\d+x\d+x\d+)?", line)
        if m and fn:
            hist[fn][m.group(1)] += 1
            if m.group(2):                       # tensor-core MMA shape (DMMA.8x8x4, DMMA.16x8x4, ...)
                hist[fn][m.group(1) + m.group(2)] += 1
    for fn, h in hist.items():
        total = sum(v for k, v in h.items() if "." not in k)
        keys = " ".join(f"{k}={h[k]}" for k in KEY if h.get(k))
        print(f"  {fn[:70]:70s} {total:6d} instr  {keys}")
