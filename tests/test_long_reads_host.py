"""Long units on the host: the segmented chains and their join (seg_chain / seg_join, cf_logic.h) give exactly the hits of the
scalar greedy search, and post_search_long, which skips the pairs that cannot meet, gives exactly post_search's lists.  The
same code runs in the long-unit kernels (k_long_seg, k_long_join, k_long_post)."""
import ctypes as C
import lzma
import os
import subprocess

import numpy as np
import pytest

import util

HIT = np.dtype([("top", "<u8"), ("bot", "<u8"), ("bwoff", "<u4"), ("len", "<u4")])


@pytest.fixture(scope="module")
def lr():
    so = os.path.join(util.CACHE, "liblongread_host.so")
    src = os.path.join(util.ROOT, "tests", "native", "longread_host.cpp")
    deps = [src, os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_logic.h"), os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_index.cpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        os.makedirs(util.CACHE, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src, deps[2]])
    lib = C.CDLL(so)
    lib.lr_load.restype = C.c_void_p
    lib.lr_chains.restype = C.c_ulonglong
    h = lib.lr_load(util.golden_index("adv").encode())
    assert h
    yield lib, C.c_void_p(h)
    lib.lr_free(C.c_void_p(h))


def pieces():
    fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
    if not os.path.exists(fa):
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa, "wb") as g:
            g.write(f.read())
    return [util.ASC2DNA[a] for _, a in util.parse_reads(fa) if len(a) >= 60]


def chimera(parts, length, seed, n_at=(), nrate=0.0):
    """Pieces of indexed reads from both strands, joined to `length` codes; Ns at the given positions and at random."""
    rng = np.random.default_rng(seed)
    out, have = [], 0
    while have < length:
        p = parts[int(rng.integers(len(parts)))]
        if rng.random() < 0.5:
            p = (3 - p)[::-1]
        out.append(p); have += len(p)
    r = np.concatenate(out)[:length].astype(np.uint8)
    if nrate:
        r[rng.random(length) < nrate] = 4
    for q in n_at:
        r[max(q, 0):q + 3] = 4
    return np.ascontiguousarray(r)


def chains(lr, read, strand, seg, min_hitlen=22):
    lib, h = lr
    n = len(read)
    a = np.zeros(n + 2, dtype=HIT); b = np.zeros(n + 2, dtype=HIT)
    na = C.c_uint32(); nb = C.c_uint32()
    re = lib.lr_chains(h, min_hitlen, read.ctypes.data_as(C.c_void_p), C.c_uint32(n), strand, C.c_uint32(seg),
                       a.ctypes.data_as(C.c_void_p), C.byref(na), b.ctypes.data_as(C.c_void_p), C.byref(nb))
    return a[:na.value], b[:nb.value], re


@pytest.mark.parametrize("seg", [7, 64, 1000, 4096])
def test_joined_segments_equal_the_scalar_chain(lr, seg):
    parts = pieces()
    total_re = 0
    for k, length in enumerate((3000, 20011, 70000)):
        read = chimera(parts, length, 100 + k, nrate=0.001)
        for strand in (0, 1):
            for mh in (15, 22):
                a, b, re = chains(lr, read, strand, seg, mh)
                assert len(a) > 0 and np.array_equal(a, b), (length, strand, mh)
                total_re += re
    assert total_re > 0          # some segments' speculative chains missed the true one and the join searched itself


def test_ns_at_segment_boundaries(lr):
    parts = pieces()
    seg = 512
    bounds = [k * seg + d for k in range(1, 40) for d in (-2, -1, 0, 1)]
    read = chimera(parts, 40 * seg + 77, 7, n_at=bounds)
    for strand in (0, 1):
        a, b, _ = chains(lr, read, strand, seg)
        assert np.array_equal(a, b)


def test_a_segment_that_never_meets_the_true_chain(lr):
    """Seg = 3: the speculative chain of a segment that starts inside a hit of the true chain reaches no position the true chain
    visits before the segment ends, so the join searches that segment itself."""
    parts = pieces()
    read = chimera(parts, 5000, 11)
    for strand in (0, 1):
        a, b, re = chains(lr, read, strand, 3)
        assert np.array_equal(a, b)
        assert re > len(a) // 4


def post(lr, read, F, R, pruned, khits=5, min_hitlen=22):
    lib, h = lr
    F = F.copy(); R = R.copy()
    lib.lr_post(h, khits, min_hitlen, read.ctypes.data_as(C.c_void_p), C.c_uint32(len(read)), F.ctypes.data_as(C.c_void_p),
                C.c_uint32(len(F)), R.ctypes.data_as(C.c_void_p), C.c_uint32(len(R)), pruned)
    return F, R


@pytest.mark.parametrize("min_hitlen", [15, 22])
def test_pruned_extension_equals_post_search_on_chains(lr, min_hitlen):
    parts = pieces()
    lib, _ = lr
    for k, length in enumerate((500, 5000, 30000, 61000)):
        read = chimera(parts, length, 300 + k, nrate=0.0005)
        F, _, _ = chains(lr, read, 0, 4096, min_hitlen)
        R, _, _ = chains(lr, read, 1, 4096, min_hitlen)
        assert lib.lr_is_chain(F.ctypes.data_as(C.c_void_p), C.c_uint32(len(F)), C.c_uint32(length)) == 1
        for khits in (1, 5):
            want = post(lr, read, F, R, 0, khits, min_hitlen)
            got = post(lr, read, F, R, 1, khits, min_hitlen)
            assert np.array_equal(want[0], got[0]) and np.array_equal(want[1], got[1]), (length, khits)
            assert not (np.array_equal(want[0], F) and np.array_equal(want[1], R)) or length < 1000


def test_reverse_complement_repeats(lr):
    """Reads made of pieces followed by their own reverse complement: the forward and reverse chains cover the same stretches,
    so nearly every F hit overlaps R hits, extensions and twins occur, and the pruned loops must find exactly those pairs."""
    lib, _ = lr
    parts = pieces()
    rng = np.random.default_rng(21)
    for k in range(6):
        out = []
        while sum(len(x) for x in out) < 8000:
            p = parts[int(rng.integers(len(parts)))][:int(rng.integers(40, 200))]
            out += [p, (3 - p)[::-1]]
        read = np.ascontiguousarray(np.concatenate(out).astype(np.uint8))
        for mh in (15, 22):
            F, _, _ = chains(lr, read, 0, 4096, mh)
            R, _, _ = chains(lr, read, 1, 4096, mh)
            assert lib.lr_is_chain(R.ctypes.data_as(C.c_void_p), C.c_uint32(len(R)), C.c_uint32(len(read))) == 1
            for khits in (1, 5):
                want = post(lr, read, F, R, 0, khits, mh)
                got = post(lr, read, F, R, 1, khits, mh)
                assert np.array_equal(want[0], got[0]) and np.array_equal(want[1], got[1]), (k, mh, khits)
                assert (want[0]["bwoff"] == 0xffffffff).any() or not np.array_equal(want[0], F)     # twins removed or hits extended
