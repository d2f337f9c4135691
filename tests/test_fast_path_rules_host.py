"""The rank16 search path's information loss, on the host.  k_search_t stores hits the death bitmap of the K-mer table ends
without their SA range (kUnk, size 0), and with --min-hitlen >= 22 it stores only the hits of at least 22 bases; load_unit
empties strand lists without a hit of min_hitlen bases, and k_prep regenerates full lists and recomputes kUnk ranges where they
can matter.  tests/native/fastpath_host.cpp degrades the scalar search's exact lists the same way and applies the same rules
(cf_logic.h: list_dropped, list_needs_regen, list_needs_exact_ranges); its records must equal the oracle's at every -k and
--min-hitlen around the boundaries the rules depend on: 16/17 (the restart increment), 21/22/23 (the 22-base class of
compareBWTHits, below which counted hits mix with uncounted short ones)."""
import ctypes as C
import functools
import lzma
import os
import subprocess

import numpy as np
import pytest

import util
from test_gpu_parity import assert_same

INDEXES = ["example", "adv", "adv_t1o2", "adv_t6o0", "adv_t8o7"]
MIN_HITLENS = [15, 16, 17, 18, 21, 22, 23, 30]
KHITS = [1, 2, 5]


@pytest.fixture(scope="module")
def lib():
    so = os.path.join(util.CACHE, "libfastpath_host.so")
    src = os.path.join(util.ROOT, "tests", "native", "fastpath_host.cpp")
    deps = [src, os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_logic.h"), os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_index.cpp"),
            os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_index.h")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        os.makedirs(util.CACHE, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so + ".tmp", src, deps[2]])
        os.replace(so + ".tmp", so)
    return C.CDLL(so)


def fast_path(lib, name, degrade=1):
    """fp_classify through the oracle's driver: the rank16 path's lists (degrade = 1) or the exact ones (0)."""
    fp = util._Classifier(lib, lib.fp_load, lib.fp_free, lib.fp_classify, util.golden_index(name))
    lib.fp_set_degrade(C.c_void_p(fp.h), degrade)
    return fp


def revcomp(a):
    return np.frombuffer(a.tobytes()[::-1].translate(bytes.maketrans(b"ACGTN", b"TGCAN")), dtype=np.uint8)


@functools.lru_cache(None)
def read_sets(name):
    """SE reads; PE reads whose mate 2 is mate 1's reverse complement (both strands of both mates in play) or another read."""
    if name == "example":
        rs = [a for _, a in util.parse_reads(os.path.join(util.GOLDEN, "example.reads.fa"))]
    else:
        fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
        if not os.path.exists(fa):
            os.makedirs(os.path.dirname(fa), exist_ok=True)
            with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa + ".tmp", "wb") as g:
                g.write(f.read())
            os.replace(fa + ".tmp", fa)
        rs = [a for _, a in util.parse_reads(fa)][::4]
    n = len(rs)
    pairs = [(rs[i], revcomp(rs[i]) if i % 2 == 0 else rs[(i * 7 + 3) % n]) for i in range(n)]
    return {"se": util.Batch(rs), "pe": util.Batch([x for x, _ in pairs], [y for _, y in pairs])}


@functools.lru_cache(None)
def oracle_records(name, rs, opt):
    o = util.Oracle(util.golden_index(name))
    on, orec, _ = o.classify(read_sets(name)[rs], util.make_oparams(**dict(opt)))
    o.close()
    return on, orec


def check(lib, name, opts):
    """Every (read set, options) case: the degraded lists' records equal the oracle's.  Returns the summed statistics."""
    fp = fast_path(lib, name)
    total = np.zeros(16, dtype=np.int64)
    try:
        for opt in opts:
            for rs, b in read_sets(name).items():
                gn, grec, st = fp.classify(b, util.make_oparams(**dict(opt)))
                on, orec = oracle_records(name, rs, opt)
                try:
                    assert_same(on, orec, gn, grec)
                except AssertionError as e:
                    raise AssertionError("%s %s %s: the rank16 path's lists give other records than the oracle: %s" % (name, rs, dict(opt), e))
                total += np.array(st, dtype=np.int64)
    finally:
        fp.close()
    return total


@pytest.mark.parametrize("min_hitlen", MIN_HITLENS)
@pytest.mark.parametrize("name", INDEXES)
def test_degraded_lists_give_the_oracle_records(lib, name, min_hitlen):
    st = check(lib, name, [(("k", k), ("min_hitlen", min_hitlen)) for k in KHITS])
    if name == "example":          # 12 reads that match the index end to end: nothing for the rules to restore
        return
    fp = fast_path(lib, name)
    K = lib.fp_kmer_chars(C.c_void_p(fp.h))
    fp.close()
    if min_hitlen >= K + 3:
        assert st[0] > 0, st[:8]               # the bitmap is in play: hits lose their range
    if min_hitlen >= 22:
        assert st[1] > 0 and st[3] > 0, st[:8]     # short hits not stored, and lists regenerated
    assert st[4] > 0 and (st[2] > 0 or min_hitlen >= 22), st[:8]    # lists given exact ranges; lists without a long hit emptied


def test_ranked_option(lib):
    for name in ("adv", "adv_t6o0"):
        check(lib, name, [(("k", 1), ("min_hitlen", 15), ("rank_slot", 2)), (("rank_slot", 2),)])


def test_exact_mode_is_the_oracle(lib):
    """degrade = 0 runs the exact lists through the same code: the baseline the degraded runs are held to."""
    fp = fast_path(lib, "adv_t1o2", degrade=0)
    try:
        for rs, b in read_sets("adv_t1o2").items():
            gn, grec, st = fp.classify(b, util.make_oparams(k=1, min_hitlen=15))
            assert_same(*oracle_records("adv_t1o2", rs, (("k", 1), ("min_hitlen", 15))), gn, grec)
            assert st[0] == 0 and st[5] == 0
    finally:
        fp.close()


ROWS_SAME_TS = 1 << 58
ROW_START = 1 << 63


def ts_case(lib, min_hitlen, blank, restore):
    rows = np.zeros(16, dtype=np.uint64)
    needs = (C.c_int * 2)()
    n = lib.fp_ts_case(min_hitlen, blank, restore, rows.ctypes.data_as(C.c_void_p), C.c_uint32(len(rows)), needs)
    assert n >= 0
    heads = [int(r) for r in rows[:n] if int(r) & ROW_START]
    return heads, list(needs)


def test_time_stamp_case(lib):
    """Mate 1's list ends through its `break`; mate 2's first counted hit (18 bases) shares its time stamp only when it sorts
    to index 0.  Its list's uncounted 12-base hit sorts behind it with its true range (3 rows / 12 bases > 1 / 18), ahead of it
    as kUnk (size 0): so the list needs its exact ranges, and with them the rows are the exact lists' rows."""
    exact, needs = ts_case(lib, 15, 0, 0)
    assert len(exact) == 2 and (exact[0] >> 40) & 0xffff == 30 and (exact[1] >> 40) & 0xffff == 18
    assert not exact[0] & ROWS_SAME_TS and exact[1] & ROWS_SAME_TS
    assert needs == [0, 1]                      # the 30-base list needs nothing; the one with a counted 18-base hit does
    blanked, _ = ts_case(lib, 15, 1, 0)
    assert len(blanked) == 2 and not blanked[1] & ROWS_SAME_TS      # the quirk: kUnk moves the counted hit off index 0
    restored, _ = ts_case(lib, 15, 1, 1)
    assert restored == exact
    # with --min-hitlen 18 the 18-base hit is not counted and the list needs no ranges (nor has it any rows to plan)
    heads, needs = ts_case(lib, 18, 1, 0)
    assert needs == [0, 0] and len(heads) == 1
