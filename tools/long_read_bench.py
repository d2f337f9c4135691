#!/usr/bin/env python3
"""Long reads through the C ABI on one GPU: a nanopore-like batch of long units only (lengths spread over 60-500 kb, ~7 %
substitutions, some Ns, a few 1 Mb reads) on a syn_big-class index, so that the time is the long-unit kernels' (reads of
1-60 kb take the short kernels and are left out).  Prints one JSON line: the card and its power limit, bases/s and reads/s, the batch
time with and without its single longest read, and the share of partial searches the segment join ran again."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def nanopore_reads(seqs, n, n_mb, seed):
    rng = np.random.default_rng(seed)
    lens = np.exp(rng.uniform(np.log(60001), np.log(500000), n)).astype(np.int64)
    lens = np.concatenate([lens, np.full(n_mb, 1000000)])
    out = []
    for L in lens:
        parts, have = [], 0
        while have < L:
            s = seqs[int(rng.integers(len(seqs)))]
            k = int(min(L - have, len(s), rng.integers(20000, 300000)))
            p = int(rng.integers(0, len(s) - k + 1))
            piece = s[p:p + k].copy()
            if rng.random() < 0.5:
                piece = (3 - piece)[::-1]
            parts.append(piece); have += k
        r = np.concatenate(parts)
        m = rng.random(L) < 0.07
        r[m] = (r[m] + rng.integers(1, 4, int(m.sum())).astype(np.uint8)) & 3
        a = np.frombuffer(b"ACGT", dtype=np.uint8)[r].copy()
        a[rng.random(L) < 0.001] = ord("N")
        out.append(a)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=40)
    ap.add_argument("--mb-reads", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import util
    from centrifuge_b200 import capi as m
    from test_gpu_parity import to_cbatch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    base = util.build_index("syn_big", 10, 10, 300000, seed=3)
    seqs = util.synth.make_genomes(10, 10, 300000, 3)
    reads = nanopore_reads(seqs, args.reads, args.mb_reads, 17)
    longest = int(np.argmax([len(a) for a in reads]))
    full = util.Batch(reads)
    rest = util.Batch([a for i, a in enumerate(reads) if i != longest])
    ix = m.Index(base, 0); ctx = m.Context(ix)

    def timed(b):
        cb = to_cbatch(b)
        ctx.classify(cb)                        # warm-up: buffers grow once
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter(); ctx.classify(cb); ts.append(time.perf_counter() - t0)
        return min(ts)

    st0 = (C.c_uint64 * 4)(); m.lib().cfb_ctx_long_stats(ctx.h, st0)
    t_full = timed(full)
    st1 = (C.c_uint64 * 4)(); m.lib().cfb_ctx_long_stats(ctx.h, st1)
    t_rest = timed(rest)
    one = timed(util.Batch([reads[longest]]))
    bases = int(sum(len(a) for a in reads))
    res = {"gpu": gpu, "reads": len(reads), "bases": bases, "batch_s": t_full, "bases_per_s": bases / t_full, "reads_per_s": len(reads) / t_full,
           "batch_without_longest_s": t_rest, "longest_read_bases": len(reads[longest]), "longest_read_alone_s": one,
           "researched_fraction": (st1[3] - st0[3]) / max(1, st1[2] - st0[2])}
    print(json.dumps(res))
    ctx.close(); ix.close()


if __name__ == "__main__":
    main()
