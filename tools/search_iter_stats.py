#!/usr/bin/env python3
"""How k_search_t spends a loop trip, from the counting instantiation's own counters (CFB_COUNT=2), on N bench reads over
the bench index; then the random-gather rate of the rank16 array with as many requests in flight per SM as the search
kernel has walks (8 CTAs x 128 threads, one and two requests per thread) next to the ceiling probe's 8192.
usage: search_iter_stats.py [n_reads] [bench.py options]"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 2000000
sys.argv = ["bench.py"] + [x for x in sys.argv[1:] if not x.isdigit()]
a = bench.parse_args()
try:
    print("card: " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True, timeout=30).stdout.strip())
except (OSError, subprocess.SubprocessError):
    print("card: nvidia-smi not available")
base, _ = bench.get_index(a)
rd = bench.make_reads(a, n, 1000)
bases, offs, lens, fl = rd.byte_form(lambda s, t: np.zeros(s, dtype=t))
ix = capi.Index(base, 0)
b = capi.make_batch(bases, offs[0], lens[0], offs[1] if a.paired else None, lens[1] if a.paired else None, fl)

ctx = capi.Context(ix)
d = ctx.upload(b)
acc = np.zeros(5)
for it in range(5):
    ms, _ = ctx.classify_resident(d)
    if it >= 2:
        acc += np.array(ms)
search_ms = acc[0] / 3
ctx.close()

os.environ["CFB_COUNT"] = "2"
ctx = capi.Context(ix)
ctx.classify(b)
req, st = ctx.requests(), ctx.search_iter_stats()
ctx.close()
del os.environ["CFB_COUNT"]

tot = sum(req.values())
wi = max(1, st["warp_iters"])
clk = st["clk_head"] + st["clk_wait"] + st["clk_tail"]
print("reads %d, timed search kernel %.3f ms, table requests %d (%.1f per read, %.2f G/s in the timed kernel)" % (n, search_ms, tot, tot / n, tot / search_ms / 1e6))
print("requests by table: %s" % req)
print("warp-iterations %d; lanes with a request per warp-iteration %.2f of 32" % (st["warp_iters"], st["lane_requests"] / wi))
print("consumer branches with a lane per warp-iteration %.2f; restart blocks with a lane per warp-iteration %.2f" % (st["consumer_paths"] / wi, st["restart_paths"] / wi))
print("warp-iterations in which a lane received a task: %.3f" % (st["task_iters"] / wi))
print("SM clocks per warp-iteration in the counting kernel: %.0f = loop top to fetch issue %.0f (%.1f %%) + wait for the loads %.0f (%.1f %%) + consume and restart %.0f (%.1f %%)"
      % (clk / wi, st["clk_head"] / wi, 100.0 * st["clk_head"] / max(1, clk), st["clk_wait"] / wi, 100.0 * st["clk_wait"] / max(1, clk), st["clk_tail"] / wi, 100.0 * st["clk_tail"] / max(1, clk)))
for ctas, ilp in ((8, 1), (8, 2), (16, 4)):
    g = [capi.gather_rate(ix, 0, 1 << 30, ctas, ilp)[0] for _ in range(3)]
    print("rank16 gather probe, %d CTAs x 128 threads x %d per thread = %d requests in flight per SM: %.2f G requests/s (min %.2f, max %.2f)"
          % (ctas, ilp, ctas * 128 * ilp, sorted(g)[1], min(g), max(g)))
ix.close()
