"""The compact rank layout on the host: the decode of cf_logic.h (cr_lf / cr_bwt), applied to half-sides converted in place from
the file's sides (cr_sb_entry / cr_convert_side), gives the oracle's LF and BWT for every row and base of the fixture indexes, at
the product's superblock span and at spans of 384 to 1536 rows that put many superblock boundaries inside them.  The layout choice
(choose_rank_layout) is checked at its edges.  The same code runs in the loader's conversion kernels and in every device reader."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import util

INDEXES = ["example", "adv", "adv_t1o2", "adv_t6o0", "adv_t8o7"]
SPANS = [1, 2, 3, 24]          # log2 half-sides per superblock: 384, 768, 1536 rows, and the product's 3.2 G rows


@pytest.fixture(scope="module")
def ch():
    so = os.path.join(util.CACHE, "libcompact_host.so")
    src = os.path.join(util.ROOT, "tests", "native", "compact_host.cpp")
    deps = [src, os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_logic.h"), os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_index.cpp")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        os.makedirs(util.CACHE, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src, deps[2]])
    lib = C.CDLL(so)
    lib.ch_load.restype = C.c_void_p
    for f in ("ch_rows", "ch_num_sides", "ch_zoff", "ch_rank16_bytes", "ch_cr_bytes"):
        getattr(lib, f).restype = C.c_uint64
    lib.ch_rank16_bytes.argtypes = lib.ch_cr_bytes.argtypes = [C.c_uint64]
    lib.ch_check.restype = C.c_longlong
    lib.ch_choose.argtypes = [C.c_uint64] * 5 + [C.c_int]
    return lib


@pytest.mark.parametrize("span", SPANS)
@pytest.mark.parametrize("name", INDEXES)
def test_compact_lf_and_bwt_match_the_oracle_on_every_row(ch, name, span):
    util.ensure_oracle()
    base = util.golden_index(name)
    h = ch.ch_load(base.encode())
    assert h
    o = util.Oracle(base)
    try:
        rows, nsides, zoff = ch.ch_rows(C.c_void_p(h)), ch.ch_num_sides(C.c_void_p(h)), ch.ch_zoff(C.c_void_p(h))
        assert nsides * 384 > rows                     # the last side is padded (A): its tail is never counted
        if span == 1 or name != "example":
            assert (2 * nsides + 1) >> min(span, 3) >= 2, (name, span)      # superblock boundaries inside the index
        first = C.c_uint64(0)
        bad = ch.ch_check(C.c_void_p(h), span, C.cast(o.lib.cfo_lf, C.c_void_p), C.cast(o.lib.cfo_bwt_char, C.c_void_p), C.c_void_p(o.h), C.byref(first))
        assert bad == 0, (name, span, bad, first.value, rows, zoff)
    finally:
        o.close()
        ch.ch_free(C.c_void_p(h))


def test_index_view_takes_the_compact_layout(ch):
    """lf_scalar / bwt_char of an IndexView whose cr is set (the scalar LF the device's extension search and test hooks run)."""
    util.ensure_oracle()
    base = util.golden_index("adv")
    h = ch.ch_load(base.encode())
    o = util.Oracle(base)
    o.lib.cfo_lf.restype = C.c_uint64
    o.lib.cfo_bwt_char.restype = C.c_int
    try:
        n = ch.ch_rows(C.c_void_p(h))
        rng = np.random.default_rng(5)
        rows = np.concatenate([np.arange(0, 2000), rng.integers(0, n, size=20000)]).astype(np.uint64)
        chars = rng.integers(0, 5, size=len(rows)).astype(np.uint8)
        out = np.zeros(len(rows), dtype=np.uint64)
        ch.ch_view_lf(C.c_void_p(h), rows.ctypes.data_as(C.c_void_p), chars.ctypes.data_as(C.c_void_p), C.c_uint64(len(rows)), out.ctypes.data_as(C.c_void_p))
        for i in range(len(rows)):
            r = C.c_uint64(int(rows[i]))
            c = int(chars[i]) if chars[i] < 4 else o.lib.cfo_bwt_char(C.c_void_p(o.h), r)
            assert int(out[i]) == o.lib.cfo_lf(C.c_void_p(o.h), r, C.c_int(c)), (i, int(rows[i]), c)
    finally:
        o.close()
        ch.ch_free(C.c_void_p(h))


def test_layout_bytes(ch):
    assert ch.ch_rank16_bytes(1000) == (6000 + 1) * 64        # 1 byte per row
    assert ch.ch_cr_bytes(1000) == 1000 * 128 + 64           # the sides themselves: 1/3 byte per row, plus the sentinel half-side


@pytest.mark.parametrize("force", [0, 1])
def test_layout_choice_at_its_edges(ch, force):
    N, sample, fixed, head = 10 ** 6, 3 * 10 ** 7, 5 * 10 ** 6, 12 << 30
    r16 = N * 128 + ch.ch_rank16_bytes(N) + sample + fixed + head        # transient sides + rank16 + the rest
    cr = ch.ch_cr_bytes(N) + sample + fixed + head

    def choose(free):
        return ch.ch_choose(free, N, sample, fixed, head, force)
    assert cr < r16
    assert choose(r16) == (1 if force else 0)                 # rank16 exactly fits
    assert choose(r16 - 1) == 1                               # rank16 exactly does not: compact
    assert choose(cr) == 1                                    # compact exactly fits
    assert choose(cr - 1) == -1                               # nothing fits
    assert choose(1 << 62) == (1 if force else 0)
    assert ch.ch_choose(r16, N, sample, fixed + 1, head, force) == 1
    assert ch.ch_choose(cr, N, sample + 1, fixed, head, force) == -1
