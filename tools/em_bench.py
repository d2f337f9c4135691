#!/usr/bin/env python3
"""Time the abundance EM (SURVEY.md 8f rank 3) on a flattened tie-set table of nt-class size: device iteration
(cfb_em_abundance) next to the host iteration the product uses for small tables (cfb_em_abundance_host), same table,
and check that the two produce the same doubles and iteration counts.  usage: em_bench.py [n_species] [n_keys] [skew]
skew (default 0): the share of keys that also name species 0, whose incidence list one device thread walks."""
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from centrifuge_b200 import capi  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 20000
K = int(sys.argv[2]) if len(sys.argv) > 2 else 400000
rng = np.random.default_rng(7)
sz = rng.integers(1, 6, size=K)
key_off = np.concatenate([[0], np.cumsum(sz)]).astype(np.uint64)
# reads tie within "genera" of 10 neighbouring species, as in the synthetic index
g = rng.integers(0, n // 10, size=K)
target = (np.repeat(g, sz) * 10 + rng.integers(0, 10, size=int(sz.sum()))).astype(np.uint32)
skew = float(sys.argv[3]) if len(sys.argv) > 3 else 0.0
if skew > 0:
    extra = rng.random(K) < skew                      # these keys get species 0 as one more target, at their end
    ends = key_off[1:].astype(np.int64)
    target = np.insert(target, ends[extra], 0).astype(np.uint32)
    key_off = np.concatenate([[0], np.cumsum(sz + extra)]).astype(np.uint64)
count = rng.integers(1, 2000, size=K).astype(np.uint64)
length = rng.integers(500000, 8000000, size=n).astype(np.uint64)
p0 = rng.random(n); p0 /= p0.sum()
lib = capi.lib()
ptr = lambda a, t: a.ctypes.data_as(C.POINTER(t))   # noqa: E731
res = {}
for name, fn, dev in (("device", lib.cfb_em_abundance, True), ("host", lib.cfb_em_abundance_host, False)):
    p = p0.copy(); iters = C.c_uint64(); diff = C.c_double()
    args = [C.c_uint64(n), C.c_uint64(K), ptr(count, C.c_uint64), ptr(key_off, C.c_uint64), ptr(target, C.c_uint32), ptr(length, C.c_uint64), ptr(p, C.c_double), C.byref(iters), C.byref(diff)]
    if dev:
        args = [C.c_int(0)] + args
        fn(*([C.c_int(0)] + [C.c_uint64(8), C.c_uint64(1), ptr(count, C.c_uint64), ptr(np.array([0, 1], dtype=np.uint64), C.c_uint64), ptr(target, C.c_uint32), ptr(length, C.c_uint64), ptr(p0.copy()[:8] / p0[:8].sum(), C.c_double), C.byref(iters), C.byref(diff)]))   # context warm-up
    t0 = time.time()
    rc = fn(*args)
    dt = time.time() - t0
    assert rc == 0, rc
    res[name] = (p, int(iters.value), float(diff.value), dt)
    print("%-6s EM: %d species, %d keys, %d contributions: %d iterations in %.3f s (%.2f ms per iteration), final diff %.3e" % (
        name, n, K, len(target), iters.value, dt, 1000 * dt / max(1, iters.value), diff.value))
same = np.array_equal(res["device"][0].view(np.uint64), res["host"][0].view(np.uint64)) and res["device"][1] == res["host"][1]
print("device and host doubles identical: %s; speed-up %.1fx" % (same, res["host"][3] / res["device"][3]))
sys.exit(0 if same else 1)
