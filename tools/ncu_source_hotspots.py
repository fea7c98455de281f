#!/usr/bin/env python
"""Source lines of one kernel ranked by warp-stall samples, from an `ncu --set full --import-source on` report:
    ncu -i X.ncu-rep --page source --csv --print-source cuda,sass --kernel-name regex:NAME --launch-count 1 > src.csv
    python tools/ncu_source_hotspots.py src.csv [top N] > hotspots_NAME.txt
(the sample attributed to the instruction after a barrier is the time spent waiting AT the barrier)."""
import collections, csv, sys
rows = list(csv.reader(open(sys.argv[1])))
top = int(sys.argv[2]) if len(sys.argv) > 2 else 30
hdr_i = next(i for i, r in enumerate(rows) if r and r[0] == "Line No")
hdr = rows[hdr_i]
i_s = hdr.index("Warp Stall Sampling (All Samples)"); i_e = hdr.index("Instructions Executed")
print(rows[1][1] if len(rows) > 1 and len(rows[1]) > 1 else "")
agg, tot = collections.OrderedDict(), 0
for r in rows[hdr_i + 1:]:
    if len(r) > max(i_s, i_e) and r[0] != "" and r[2] == "-":
        try: ln, s, ie = int(r[0]), int(r[i_s]), int(r[i_e])
        except ValueError: continue
        a = agg.setdefault(ln, [r[1], 0, 0]); a[1] += s; a[2] += ie; tot += s
print(f"total stall samples {tot}")
for ln, (src, s, ie) in sorted(agg.items(), key=lambda x: -x[1][1])[:top]:
    print(f"{ln:5d} {100.0 * s / max(1, tot):5.1f} %  {ie:9d} instr  {src.strip()[:150]}")
