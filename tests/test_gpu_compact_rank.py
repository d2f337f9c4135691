"""The compact rank layout on the device (1/3 byte per BWT row, chosen at load when rank16 does not fit, or forced with
CFB_RANK16=0): the LF and resolve hooks, the records through the C ABI (equal to the default layout's and to the oracle's),
centrifuge-class against the reference's recorded digests, the big indexes, and the automatic choice under memory pressure."""
import ctypes as C
import functools
import lzma
import os
import re
import subprocess

import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu

INDEXES = ["example", "adv", "adv_t1o2", "adv_t6o0", "adv_t8o7"]
EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
BIG = pytest.mark.skipif(os.environ.get("CFB_TEST_SKIP_BIG") == "1", reason="CFB_TEST_SKIP_BIG=1")
KNOBS = ("CFB_RANK16", "CFB_FTABK", "CFB_FTABD", "CFB_RESOLVE_TABLE", "CFB_WALK8", "CFB_WALK8_ROWS", "CFB_KEEP_SHORT", "CFB_COUNT", "CFB_HBM_HEADROOM_GB")


def capi():
    from centrifuge_b200 import capi as m
    return m


def set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def revcomp(a):
    return np.frombuffer(a.tobytes()[::-1].translate(bytes.maketrans(b"ACGTN", b"TGCAN")), dtype=np.uint8)


def reads_of(name):
    fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
    if name == "example":
        fa = os.path.join(util.GOLDEN, "example.reads.fa")
    elif not os.path.exists(fa):
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa, "wb") as g:
            g.write(f.read())
    return [a for _, a in util.parse_reads(fa)]


@functools.lru_cache(None)
def read_sets(name):
    """SE, PE with twins, mixed lengths across every read-length class (joined reads up to ~900 bases), and long units of more
    than 60 000 bases (single and as mate 2)."""
    rs = reads_of(name)
    rng = np.random.default_rng(len(name))
    se = rs[:1500]
    prs = [(rs[i], revcomp(rs[i]) if i % 3 == 0 else rs[(i * 7 + 1) % len(rs)]) for i in range(min(len(rs), 800))]
    mixed = []
    for i in range(400):
        k = int(rng.integers(1, 9))
        j = int(rng.integers(0, len(rs)))
        mixed.append(np.concatenate([rs[(j + q) % len(rs)] for q in range(k)]))
    def joined(start, n):
        out, q = [], start
        while sum(len(x) for x in out) < n:
            x = rs[q % len(rs)]; out.append(revcomp(x) if q % 2 else x); q += 1
        return np.concatenate(out)
    longs = [joined(0, 60500), joined(5, 62000)]
    return {"se": util.Batch(se), "pe": util.Batch([x for x, _ in prs], [y for _, y in prs]), "mixed": util.Batch(mixed),
            "long_se": util.Batch(longs + se[:50]), "long_mate2": util.Batch(se[:2], longs)}


def records(ix, b, **kw):
    m = capi()
    ctx = m.Context(ix, m.make_params(**kw))
    off, recs = ctx.classify(to_cbatch(b))
    ctx.close()
    return np.diff(off.astype(np.int64)).astype(np.uint32), recs


@functools.lru_cache(None)
def oracle_records(name, rs, opt):
    return oracle(util.golden_index(name), read_sets(name)[rs], **OPTS[opt])


def oracle(base, b, **kw):
    o = util.Oracle(base)
    on, orec, _ = o.classify(b, util.make_oparams(**kw))
    o.close()
    return on, orec


OPTS = {"default": {}, "k1_minhit15": {"k": 1, "min_hitlen": 15}}
TABLES = {"kmer_default": {}, "kmer_at_ftab": {"CFB_FTABK": "FC"}, "no_bitmap": {"CFB_FTABD": "0"}}


@pytest.mark.parametrize("tables", sorted(TABLES))
@pytest.mark.parametrize("name", INDEXES)
def test_compact_records_equal_rank16_and_oracle(name, tables, monkeypatch):
    m = capi()
    base = util.golden_index(name)
    sets = read_sets(name)
    set_env(monkeypatch, {})
    ix = m.Index(base, 0)
    fc = ix.info.ftab_chars
    want = {(rs, opt): records(ix, b, **OPTS[opt]) for rs, b in sets.items() for opt in OPTS}
    ix.close()
    set_env(monkeypatch, dict({k: v.replace("FC", str(fc)) for k, v in TABLES[tables].items()}, CFB_RANK16="0"))
    ix = m.Index(base, 0)
    tb = ix.tables()
    assert tb["rank16_bytes"] == 0 and tb["sides_bytes"] == ix.info.num_sides * 128 + 64, tb
    assert tb["resolve_table_bytes"] == 0 and tb["walk8_bytes"] == 0, tb
    if tables == "no_bitmap":
        assert tb["ftabd_chars"] == 0, tb
    else:
        assert tb["ftabk_bytes"] > 0 and tb["ftabd_chars"] == tb["ftabk_chars"] + 3, tb
    for (rs, opt), (wn, wrec) in want.items():
        gn, grec = records(ix, sets[rs], **OPTS[opt])
        on, orec = oracle_records(name, rs, opt)
        try:
            assert_same(on, orec, gn, grec)
        except AssertionError as e:
            raise AssertionError("%s %s %s %s: compact vs oracle: %s" % (name, tables, rs, opt, e))
        try:
            assert_same(wn, wrec, gn, grec)
        except AssertionError as e:
            raise AssertionError("%s %s %s %s: compact vs rank16: %s" % (name, tables, rs, opt, e))
    ix.close()


@pytest.mark.parametrize("name", INDEXES)
def test_compact_lf_and_resolve_hooks_match_oracle(name, monkeypatch):
    set_env(monkeypatch, {"CFB_RANK16": "0"})
    m = capi()
    base = util.golden_index(name)
    ix = m.Index(base, 0)
    n_rows = ix.info.len + 1
    rng = np.random.default_rng(3)
    edges = [0, n_rows - 1] + list(range(0, n_rows, 192)) + list(range(0, n_rows, 64))
    rows = np.array(sorted({r + d for r in edges for d in (-1, 0, 1) if 0 <= r + d < n_rows}), dtype=np.uint64)
    rows = np.concatenate([rows, rng.integers(0, n_rows, size=20000).astype(np.uint64)])
    chars = rng.integers(0, 5, size=len(rows)).astype(np.uint8)
    got, gres = m.test_lf(ix, rows, chars), m.test_resolve(ix, rows)
    ix.close()
    o = util.Oracle(base)
    o.lib.cfo_lf.restype = C.c_uint64
    o.lib.cfo_bwt_char.restype = C.c_int
    o.lib.cfo_resolve.restype = C.c_uint64
    for i in range(len(rows)):
        r, c = C.c_uint64(int(rows[i])), int(chars[i])
        if c > 3:
            c = o.lib.cfo_bwt_char(C.c_void_p(o.h), r)
        assert int(got[i]) == o.lib.cfo_lf(C.c_void_p(o.h), r, C.c_int(c)), (name, i, int(rows[i]), c)
        assert int(gres[i]) == o.lib.cfo_resolve(C.c_void_p(o.h), r, None), (name, i, int(rows[i]))
    o.close()


def test_request_counts_on_the_compact_layout(monkeypatch):
    """CFB_COUNT=2 counts the compact search's sector pieces in slot 0; CFB_COUNT=1 counts the reference's operations as on rank16."""
    m = capi()
    base = util.golden_index("adv")
    b = read_sets("adv")["se"]
    got = {}
    for layout in ("rank16", "compact"):
        set_env(monkeypatch, {"CFB_RANK16": "0"} if layout == "compact" else {})
        ix = m.Index(base, 0)
        monkeypatch.setenv("CFB_COUNT", "1")
        ctx = m.Context(ix, m.make_params()); ctx.classify(to_cbatch(b)); c1 = ctx.counters(); ctx.close()
        monkeypatch.setenv("CFB_COUNT", "2")
        ctx = m.Context(ix, m.make_params()); ctx.classify(to_cbatch(b)); req = ctx.requests(); ctx.close()
        got[layout] = (c1, req)
        if layout == "compact":
            assert req["rank16"] > 0, req
            assert m.gather_ceiling(ix, 0, 1 << 24)[0] > 0
        ix.close()
    assert got["rank16"][0] == got["compact"][0]


# ----------------------------------------------------------------------------- centrifuge-class
@pytest.fixture(scope="module")
def syn():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    seqs = util.synth.make_genomes(5, 4, 60000, 7)
    return base, seqs


def run_cli(args, tmp, tag, env):
    tsv, rep, kr = (str(tmp / (tag + x)) for x in (".tsv", ".rep", ".kr"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep, "--kreport-file", kr], stdout=subprocess.DEVNULL,
                       stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1", **env))
    assert p.returncode == 0, p.stderr.decode()
    err = p.stderr.decode()
    layout = re.search(r"index load \S+ s \((\w+) rank layout\)", err)
    assert layout, err
    out = []
    for f in (tsv, rep, kr):
        with open(f, "rb") as g:
            out.append(g.read())
    return tuple(out), layout.group(1)


def test_cli_on_the_compact_layout_gives_the_reference_bytes(syn, tmp_path):
    """The reads, options and recorded reference digests of the text operator's SE and PE cases (test_gpu_text.py), through the
    text operator and the record-level reader, with the compact layout forced; the Kraken-style report equals rank16's."""
    import test_gpu_text as tt
    base, seqs = syn
    rng = np.random.default_rng(1)
    reads = (util.synth.sample_reads(seqs, 2500, 60, seed=11, lens=(1, 120)) + util.synth.sample_reads(seqs, 2500, 150, seed=12, lens=(100, 300))
             + util.synth.sample_reads(seqs, 600, 500, seed=13, lens=(300, 900)))
    reads = tt.decorate(reads, rng)
    fq = str(tmp_path / "r.fq")
    tt.write_fq(fq, reads, rng, tail_newline=False)
    rng = np.random.default_rng(2)
    prs = util.synth.sample_pairs(seqs, 5000, 125, seed=31)
    r1 = tt.decorate([(n, x) for n, x, _ in prs], rng)
    r2 = [(n + "/2", y[: max(1, len(y) - (i % 40))]) for i, (n, _, y) in enumerate(prs)]
    f1, f2 = str(tmp_path / "p_1.fq"), str(tmp_path / "p_2.fq")
    tt.write_fq(f1, r1, rng); tt.write_fq(f2, r2, rng)
    cases = [("fastq_se/", ["-q", "-x", base, "-U", fq]), ("fastq_se/-k 1", ["-q", "-x", base, "-U", fq, "-k", "1"]),
             ("fastq_pe/", ["-q", "-x", base, "-1", f1, "-2", f2])]
    for key, args in cases:
        want = tt.run_ref(key, args, tmp_path, "ref")
        ours, lay = run_cli(args, tmp_path, "r16", {})
        assert lay == "rank16"
        for extra in ([], ["--host-parse"]):
            got, lay = run_cli(args + extra, tmp_path, "cr", {"CFB_RANK16": "0"})
            assert lay == "compact"
            util.assert_matches(got[:2], want, key, extra)
            assert got == ours, (key, extra)


# ----------------------------------------------------------------------------- big indexes
def big_vs_oracle(base, codes, monkeypatch):
    m = capi()
    set_env(monkeypatch, {"CFB_RANK16": "0", "CFB_HBM_HEADROOM_GB": "2"})
    ix = m.Index(base, 0)
    tb = ix.tables()
    assert tb["rank16_bytes"] == 0 and tb["sides_bytes"] > 0 and tb["ftabk_bytes"] > 0, tb
    b = util.Batch(list(codes))
    gn, grec = records(ix, b)
    ix.close()
    on, orec = oracle(base, b)
    assert_same(on, orec, gn, grec)
    return tb


@BIG
def test_compact_u32_sample_index_matches_oracle(monkeypatch):
    """> 65 535 sequences at 7 Gbp (u32 SA sample), 200 K reads."""
    import test_gpu_bench_config as bc
    m = capi()
    base, so = bc.synth_index("wide", 7000, 10, 100000)
    big_vs_oracle(base, m.synth_reads(so, 200000, 100, 778), monkeypatch)


@BIG
def test_compact_index_beyond_2_32_rows_matches_oracle(monkeypatch):
    """The 9 Gbp bench index: rows beyond 2^32, so more than one superblock of the compact layout, 200 K reads."""
    import test_gpu_bench_config as bc
    m = capi()
    base, so = bc.synth_index("bench", 900, 10, 1000000)
    ix = m.Index(base, -1)
    assert ix.info.len > (1 << 32)
    ix.close()
    big_vs_oracle(base, m.synth_reads(so, 200000, 100, 4244), monkeypatch)


# ----------------------------------------------------------------------------- automatic choice
NEED = re.compile(r"rank16 needs (\d+) bytes and the compact layout (\d+), each plus (\d+) bytes .*; (\d+) bytes are free")


def test_layout_is_chosen_from_free_memory(monkeypatch):
    """Device memory held with torch: with room for the compact layout but not rank16 the load takes the compact layout and gives
    the same records; with room for neither it fails with CFB_ENOMEM, naming both needs, and leaves no device memory behind."""
    import torch
    m = capi()
    base = util.build_index("syn_big", 10, 10, 300000, seed=3)
    b = util.Batch(reads_of("adv")[:1000])
    set_env(monkeypatch, {})
    ix = m.Index(base, 0)
    want = records(ix, b)
    ix.close()
    torch.cuda.synchronize()
    set_env(monkeypatch, {"CFB_HBM_HEADROOM_GB": "0"})         # the head-room term is 0: the needs are the layouts' alone
    held = []

    def hold_until(free_target):
        """hold device memory until at most free_target bytes are free (2 MB steps at the end); returns what is free"""
        while True:
            free = torch.cuda.mem_get_info()[0]
            if free <= free_target:
                return free
            step = free - free_target - (4 << 20)
            held.append(torch.empty(min(step, 1 << 30) if step > (2 << 20) else (2 << 20), dtype=torch.uint8, device="cuda"))
    try:
        # 1. room for neither: the message names both needs and the free bytes; nothing is left allocated
        hold_until(16 << 20)          # below the 10-mer tables alone
        before = torch.cuda.mem_get_info()[0]
        with pytest.raises(m.CfbError) as e:
            m.Index(base, 0)
        after = torch.cuda.mem_get_info()[0]
        assert "error -3" in str(e.value) and "fits no rank layout" in str(e.value), str(e.value)
        assert after == before
        mm = NEED.search(str(e.value))
        assert mm, str(e.value)
        need_r16, need_cr = int(mm.group(1)), int(mm.group(2))
        assert need_cr < need_r16 and need_cr > before
        # 2. room for the compact layout only
        while held:
            held.pop()
        torch.cuda.empty_cache()
        free = hold_until((need_cr + need_r16) // 2)
        if free < need_cr:        # a 2 MB step overshot: give one back
            held.pop(); torch.cuda.empty_cache()
            free = torch.cuda.mem_get_info()[0]
        assert need_cr <= free < need_r16, (need_cr, free, need_r16)
        ix = m.Index(base, 0)
        tb = ix.tables()
        assert tb["rank16_bytes"] == 0 and tb["sides_bytes"] > 0, tb
        while held:
            held.pop()
        torch.cuda.empty_cache()
        gn, grec = records(ix, b)
        ix.close()
        assert_same(want[0], want[1], gn, grec)
    finally:
        held.clear()
        torch.cuda.empty_cache()
