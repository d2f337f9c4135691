#!/usr/bin/env python3
"""Where the scoring stage behind the search spends its time, on one resident window of the bench batch (same generator, seed,
index and CFB_HBM_HEADROOM_GB as bench.py; per-taxon counters folded on the device as bench.py does):
  * each kernel from k_score to k_fold_counts (the `score_compact` stage of bench.py's kernel_ms), from torch.profiler with CUDA
    activities, averaged over several launches of the window;
  * from the counting instantiation of k_score (CFB_COUNT=2) over the same window: rows and distinct ids per unit, the units
    that enter the tree reduction and the rank rounds they run, and the warps whose rows did not fit the shared pool.
usage: score_stage_stats.py [--json FILE] [bench.py options]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

out_json = None
if "--json" in sys.argv:
    i = sys.argv.index("--json")
    out_json = sys.argv[i + 1]
    del sys.argv[i:i + 2]
sys.argv = ["bench.py"] + sys.argv[1:]
a = bench.parse_args()

import torch  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

if not torch.cuda.is_available():
    raise SystemExit("score_stage_stats.py: no CUDA device")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = "nvidia-smi not available"
print("card: " + card)

base, _ = bench.get_index(a)
rd = bench.make_reads(a, a.reads, 1000)      # bench.py's batch (rank 0), of which the first window is measured
n = rd.n
# bench.py's head-room formula, so that the loader builds the same derived tables
E2E_SLOTS = 8
lc = 128 if rd.lmax <= 128 else (160 if rd.lmax <= 160 else (320 if rd.lmax <= 320 else ((rd.lmax + 1023) // 1024) * 1024))
per_unit = rd.mates * ((lc // 22 + 2) * 48 + (lc / 4 + 8) * 48 / 32 + (lc // 32 + 1) * 24 + 3.5 * lc + 64) + 1776 + 160
headroom_gb = max(12.0, ((E2E_SLOTS * a.sub + a.chunk) * per_unit * 1.3 + float(rd.lens.sum()) + 8.0 * n * rd.mates * 2 + (3 << 30)) / 2 ** 30)
os.environ.setdefault("CFB_HBM_HEADROOM_GB", "%.1f" % headroom_gb)

win = min(a.chunk, n)
w = rd.sub(0, win)
bases, offs, lens, fl = w.byte_form(lambda s, t: np.zeros(s, dtype=t))
ix = capi.Index(base, 0)
b = capi.make_batch(bases, offs[0], lens[0], offs[1] if a.paired else None, lens[1] if a.paired else None, fl)

# ---- kernel times
ctx = capi.Context(ix)
ctx.count_records(True)
d = ctx.upload(b)
stage = np.zeros(5)
for _ in range(3):
    ctx.classify_resident(d)
REPS = 5
for _ in range(REPS):
    ms, _ = ctx.classify_resident(d)
    stage += np.array(ms)
stage /= REPS
from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(REPS):
        ctx.classify_resident(d)
    torch.cuda.synchronize()
ctx.close()

kern = [e for e in prof.events() if getattr(e, "device_type", None) is not None and str(e.device_type).endswith("CUDA")]
kern.sort(key=lambda e: e.time_range.start)
names = [e.name for e in kern]
per_name, order = {}, []
# the stage: every kernel from k_score up to the counter fold (k_cnt_commit, launched when the batch is collected, is not in it)
inside = False
for e in kern:
    nm = e.name
    if nm.startswith("void k_score") or nm.startswith("k_score"):
        inside = True
    if inside:
        key = nm.split("(")[0].split("<")[0].replace("void ", "")
        if key not in per_name:
            per_name[key] = 0.0
            order.append(key)
        t = getattr(e, "device_time", None)
        if t is None:
            t = e.cuda_time
        per_name[key] += t / 1000.0
    if "k_fold_counts" in nm:
        inside = False
print("window: %d units of the bench batch (%s); stage times by CUDA events (kernel_ms of bench.py, one window): search %.3f, "
      "prep_rows %.3f, resolve %.3f, score_compact %.3f ms" % (win, bench.describe(a), stage[0], stage[1], stage[2], stage[3]))
print("score_compact kernels by torch.profiler, ms per window (mean of %d):" % REPS)
tot = 0.0
for k in order:
    print("  %-40s %8.3f" % (k, per_name[k] / REPS))
    tot += per_name[k] / REPS
print("  %-40s %8.3f" % ("sum", tot))

# ---- distributions from the counting instantiation
os.environ["CFB_COUNT"] = "2"
cctx = capi.Context(ix)
cctx.classify(b)
st = cctx.score_stats()
cctx.close()
del os.environ["CFB_COUNT"]
ix.close()
u = max(1, st["units"])
buckets = ["1", "2-3", "4-7", "8-15", "16-31", "32-63", "64-127", ">=128"]
print("units with rows %d of %d; rows per unit %.2f; distinct ids per unit %.2f" % (st["units"], win, st["rows"] / u, st["distinct_ids"] / u))
print("rows per unit:         " + ", ".join("%s: %.2f %%" % (k, 100.0 * v / u) for k, v in zip(buckets, st["rows_hist"])))
print("distinct ids per unit: " + ", ".join("%s: %.2f %%" % (k, 100.0 * v / u) for k, v in zip(buckets, st["distinct_ids_hist"])))
print("units in the tree reduction: %.2f %% (%d), rank rounds per such unit %.2f" % (100.0 * st["reduce_units"] / u, st["reduce_units"], st["reduce_rounds"] / max(1, st["reduce_units"])))
print("k_score warps on the global scratch: %.3f %% (%d of %d warps with rows)" % (100.0 * st["warps_global"] / max(1, st["warps"]), st["warps_global"], st["warps"]))
if out_json:
    with open(out_json, "w") as f:
        json.dump({"card": card, "window": win, "stage_ms": list(stage), "kernels_ms": {k: per_name[k] / REPS for k in order}, "score_stats": st}, f, indent=1)
