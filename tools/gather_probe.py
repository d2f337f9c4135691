#!/usr/bin/env python3
"""Random-gather ceilings of this device over the bench index replica's own arrays, per table: independent 16- or 8-byte LDG
requests, the load the walk kernels use."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

sys.argv = ["bench.py"] + sys.argv[1:]
a = bench.parse_args()
base, d = bench.get_index(a)
ix = capi.Index(base, 0)
tb = ix.tables()
print("index replica: %.1f GB in HBM; tables %s" % (tb["total_bytes"] / 1e9, {k: v for k, v in tb.items() if k.endswith("chars") or k == "walk8_rows"}))
names = {0: "rank16 (16 B entries, %.1f GB)" % (tb["rank16_bytes"] / 1e9), 1: "K-mer table + death bitmap (16 B entries, %.1f GB)" % (tb["ftabk_bytes"] / 1e9),
         2: "walk8 (8 B entries, %.1f GB)" % (tb["walk8_bytes"] / 1e9), 3: "resolve table (8 B words, %.1f GB)" % (tb["resolve_table_bytes"] / 1e9)}
for t in (0, 1, 2, 3):
    try:
        g, ms = capi.gather_ceiling(ix, t, 1 << 31)
        print("LDG   %-45s %7.2f G requests/s  (%.1f ms)" % (names[t], g, ms))
    except capi.CfbError as e:
        print("LDG   %-45s not built (%s)" % (names[t], e))
ix.close()
