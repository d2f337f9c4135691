"""An index of more than 65 535 sequences (u32 sequence ids, u32 SA sample, boundary rows): 66 000 random 120-base sequences,
the second half 3 %-diverged copies of the first, 300 species in 30 genera.  test_oracle's wide-sample test builds the same
index into the same cache directory (same data, same recorded digest "wide"); wide_index() checks that the cached FASTA is the
one it would write, so the two recipes cannot drift apart unnoticed."""
import hashlib
import os

import numpy as np

import util

N, L = 66000, 120


def wide_genomes():
    """(N, L) uint8 base codes of the index's sequences"""
    rng = np.random.default_rng(44)
    g = rng.integers(0, 4, size=(N, L), dtype=np.uint8)
    g[33000:] = np.where(rng.random((33000, L)) < 0.03, (g[:33000] + 1) & 3, g[:33000])
    return g


def wide_index():
    """(index base path, sequences) of the wide index, built once into util.CACHE/wide"""
    g = wide_genomes()
    A = util.synth.ACGT
    fasta = b"".join(b">c%d\n" % i + A[g[i]].tobytes() + b"\n" for i in range(N))
    d = os.path.join(util.CACHE, "wide")
    base = os.path.join(d, "idx")
    fa = os.path.join(d, "g.fa")
    if not os.path.exists(os.path.join(d, "done")):
        os.makedirs(d, exist_ok=True)
        with open(fa, "wb") as f:
            f.write(fasta)
        with open(os.path.join(d, "conv.tsv"), "w") as f:
            for i in range(N):
                f.write("c%d\t%d\n" % (i, 1000 + i % 300))
        with open(os.path.join(d, "nodes.dmp"), "w") as f:
            f.write("1\t|\t1\t|\tno rank\t|\n")
            for t in range(30):
                f.write("%d\t|\t1\t|\tgenus\t|\n" % (100 + t))
            for t in range(300):
                f.write("%d\t|\t%d\t|\tspecies\t|\n" % (1000 + t, 100 + t % 30))
        with open(os.path.join(d, "names.dmp"), "w") as f:
            f.write("1\t|\troot\t|\t\t|\tscientific name\t|\n")
        util.build_cf([fa], os.path.join(d, "conv.tsv"), os.path.join(d, "nodes.dmp"), os.path.join(d, "names.dmp"), base, "wide")
        open(os.path.join(d, "done"), "w").close()
    with open(fa, "rb") as f:
        if hashlib.md5(f.read()).digest() != hashlib.md5(fasta).digest():
            raise AssertionError("%s holds another wide index than tests/util_wide.py describes" % d)
    return base, g
