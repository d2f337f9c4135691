#!/usr/bin/env python3
"""One classification of N bench reads on the bench index under whatever CFB_* knobs the environment sets -- the
unit of an ncu A/B capture (e.g. CFB_WALK8=0 for the search without walk8 next to the default tables).
usage: ab_probe.py [n_reads]"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from centrifuge_b200 import capi  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 500000
n = int(os.environ.get("CFB_PROBE_READS", n))
sys.argv = ["bench.py"] + sys.argv[2:]
a = bench.parse_args()
base, d = bench.get_index(a)
rd = bench.make_reads(a, n, 1000)
bases, offs, lens, fl = rd.byte_form(lambda s, t: np.zeros(s, dtype=t))
ix = capi.Index(base, 0)
ctx = capi.Context(ix)
b = capi.make_batch(bases, offs[0], lens[0], None, None, fl)
d = ctx.upload(b)
acc = np.zeros(5); reps = int(os.environ.get("CFB_PROBE_REPS", 6))
for it in range(reps):
    ms, nrec = ctx.classify_resident(d)
    if it >= 2:
        acc += np.array(ms)
ms = list(acc / max(1, reps - 2))
print("probe: %d reads, tables %s" % (n, {k: v for k, v in ix.tables().items() if k in ("ftabk_chars", "walk8_rows", "resolve_entry_bytes", "sides_bytes")}))
print("probe: kernel ms search %.3f prep %.3f resolve %.3f score %.3f total %.3f -> %.1f M reads/s" % (ms[0], ms[1], ms[2], ms[3], ms[4], n / ms[4] / 1e3))
ctx.close(); ix.close()
