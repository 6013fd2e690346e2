#!/usr/bin/env python
"""Per-level timings of one resident fit: routed entries, parent slots, route+hist time and the implied entry rate.
Tells whether a level is bound by the shared-atomic rate (constant entries/us) or by per-slot overheads (deep levels).
Also prints the fit's unique record count U and the TreePoint record format the level kernel gathered, with its footprint:
whether the record set fits the L2 decides the gather rate."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "spark-network-traffic-classifier_b200"))
import torch, bench
from b200flow import forest
a = bench.parse()
wl = bench.Workload(a)
rec, dicts = wl.make(a.rows, "cuda")
for _ in range(2):
    bench.step_resident(wl, rec, dicts, a, None)
torch.cuda.synchronize()
forest.PROFILE = {}
t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
t0.record(); _, _, st, _ = bench.step_resident(wl, rec, dicts, a, None); t1.record()
torch.cuda.synchronize()
P = forest.PROFILE
print("step %.2f ms (with per-kernel events)" % t0.elapsed_time(t1))
U, rb = st["unique_rows"], st.get("record_bytes", 0)
print("rows %d  unique records U %d  record format %s, %d bytes  footprint %.1f MB"
      % (st["rows"], U, st.get("record_format", "bytes"), rb, U * rb / 1e6))
ents = [int(e) for e in P.get("_route_entries", [])]
rt = [x.elapsed_time(y) for x, y in P.get("route_hist_level", [])]
sc = [x.elapsed_time(y) for x, y in P.get("score_level", [])]
print("level  routed_entries  route_ms  Mentries/ms  score_ms")
for i, t in enumerate(rt):
    e = ents[i] if i < len(ents) else -1
    print("%3d %14d %9.3f %10.2f %9.3f" % (i, e, t, e / t / 1e6 if t > 0 else 0, sc[i] if i < len(sc) else float("nan")))
for k, v in P.items():
    if not k.startswith("_"):
        print("%-20s %3d launches %8.3f ms" % (k, len(v), sum(x.elapsed_time(y) for x, y in v)))
