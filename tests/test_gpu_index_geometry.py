"""GPU: the builder, the loader's derived tables and the kernels on indexes built with other -t/--ftabchars and -o/--offrate
values than the default (10, 4), and on K-mer ranges past the 24-bit width the K-mer table stores.

ftabChars sets the ftab, the K the K-mer table starts from, the LF steps k_build_ftabk takes above it and when the death bitmap
applies (min_hitlen >= K + 3); offRate sets which rows k_resolve_c finds sampled.  Geometries: the committed builds of the adv
genomes at -t 6 -o 0 (every row sampled; K = 8 > ftabChars without forcing), -t 1 -o 2 (K = 8 from a 1-mer ftab) and
-t 8 -o 7 (long resolve walks; K = ftabChars, bitmap only), and the strain-rich syn_a genomes at -t 12 -o 5 (not committed:
its ftab alone is 134 MB; the test builds it and checks the recorded digest of the reference builder's files)."""
import functools
import lzma
import os
import struct
import time

import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu

GEOMETRIES = {"adv_t6o0": (6, 0), "adv_t1o2": (1, 2), "adv_t8o7": (8, 7), "syn_a_t12o5": (12, 5)}
OPTIONS = {"default": {}, "k1": dict(k=1), "minhit15": dict(min_hitlen=15), "family": dict(rank_slot=3)}
SYN_A = ("syn_a", 5, 4, 60000, 7)


def capi():
    from centrifuge_b200 import capi as m
    return m


def index_base(name):
    if name.startswith("adv_"):
        return util.golden_index(name)
    return util.build_index(*SYN_A, strains=True, ftab_chars=12, off_rate=5)


def header(base):
    """(len, offRate, ftabChars, zOff, fchr) from the .1.cf file (the bowtie2 layout the loader reads)."""
    with open(base + ".1.cf", "rb") as f:
        d = f.read()
    ln, line_rate, _, off_rate, ftab_chars, _ = struct.unpack_from("<QiiiiI", d, 4)
    p = 4 + 8 + 20
    npat = struct.unpack_from("<Q", d, p)[0]; p += 8 + 8 * npat
    nfrag = struct.unpack_from("<Q", d, p)[0]; p += 8 + 24 * nfrag
    side = 1 << line_rate
    p += (ln // 4 + 1 + side - 33) // (side - 32) * side
    zoff = struct.unpack_from("<Q", d, p)[0]
    fchr = struct.unpack_from("<5Q", d, p + 8)
    return ln, off_rate, ftab_chars, zoff, fchr


def kmer_k(ftab_chars, length):
    """The loader's K for the K-mer table: from ftabChars up while K < 15 and 4^(K+1) <= len/4."""
    k = ftab_chars
    while k < 15 and 4 ** (k + 1) <= length // 4:
        k += 1
    return k


@functools.lru_cache(None)
def genomes(name):
    if name.startswith("adv_"):
        d = os.path.join(util.CACHE, "adv_genomes")
        if not os.path.exists(os.path.join(d, "genomes.fa")):
            util.synth.write_adversarial(d, seed=33, n_reads=10)
        return [util.ASC2DNA[a] & 3 for _, a in util.parse_reads(os.path.join(d, "genomes.fa"))]
    return util.synth.make_genomes(*SYN_A[1:])


def revcomp(a):
    return np.frombuffer(a.tobytes()[::-1].translate(bytes.maketrans(b"ACGTN", b"TGCAN")), dtype=np.uint8)


@functools.lru_cache(None)
def read_sets(name):
    fc = GEOMETRIES[name][0]
    seqs = genomes(name)
    k = kmer_k(fc, header(index_base(name))[0])
    sets = {}
    if name.startswith("adv_"):
        fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa, "wb") as g:
            g.write(f.read())
        sets["adv"] = util.Batch([a for _, a in util.parse_reads(fa)])
    sets["se_1_300"] = util.Batch([a for _, a in util.synth.sample_reads(seqs, 3000, 100, seed=301, lens=(1, 300))])
    # an N at depth d of the first partial search: fw strand at read offset len-1-d, rc strand at offset d
    base_reads = [a for _, a in util.synth.sample_reads(seqs, 120, 90, seed=302, nrate=0, random_frac=0)]
    nreads = []
    for d in (fc - 1, fc, k, k + 2):
        for i, a in enumerate(base_reads):
            a = a.copy()
            a[len(a) - 1 - d if i % 2 == 0 else d] = ord("N")
            nreads.append(a)
    sets["n_at_ftab_and_k"] = util.Batch(nreads)
    # pairs: mate 2 is mate 1's reverse complement (every hit twice: list regeneration and twin removal), or the other end
    prs = util.synth.sample_pairs(seqs, 2000, 150, seed=303)
    sets["pe_twins"] = util.Batch([x for _, x, _ in prs], [revcomp(x) if i % 2 == 0 else y for i, (_, x, y) in enumerate(prs)])
    if name == "syn_a_t12o5":
        sets["long"] = util.Batch([a for _, a in util.synth.sample_reads(seqs, 800, 321, seed=304, lens=(321, 800))])
    return sets


@functools.lru_cache(None)
def oracle_records(name, opt, rs):
    o = util.Oracle(index_base(name))
    on, orec, _ = o.classify(read_sets(name)[rs], util.make_oparams(**OPTIONS[opt]))
    o.close()
    return on, orec


def gpu_records(ix, batch, **kw):
    m = capi()
    ctx = m.Context(ix, m.make_params(**kw))
    off, recs = ctx.classify(to_cbatch(batch))
    ctx.close()
    return np.diff(off.astype(np.int64)).astype(np.uint32), recs


def set_env(monkeypatch, env):
    for k in ("CFB_FTABK", "CFB_FTABD", "CFB_RESOLVE_TABLE", "CFB_WALK8_ROWS", "CFB_KEEP_SHORT", "CFB_COUNT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ----------------------------------------------------------------------------- builder
@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_builder_writes_the_reference_builders_bytes(name, tmp_path):
    m = capi()
    fc, orate = GEOMETRIES[name]
    d = str(tmp_path)
    if name.startswith("adv_"):
        util.synth.write_adversarial(d, seed=33, n_reads=10)
        want = [open("%s.%s.cf" % (util.golden_index(name), k), "rb").read() for k in "1234"]
    else:
        util.synth.write_genomes(d, *SYN_A[1:], strains=True)
        key = util.index_key(*SYN_A, strains=True, ftab_chars=fc, off_rate=orate)
        want = util.reference("index/" + key, lambda: [open("%s.%s.cf" % (index_base(name), k), "rb").read() for k in "1234"])
    m.build_index(m.build_opts(d + "/mine", fasta=[d + "/genomes.fa"], conversion_table=d + "/conv.tsv", taxonomy_tree=d + "/nodes.dmp",
                               name_table=d + "/names.dmp", ftab_chars=fc, off_rate=orate))
    got = [open("%s/mine.%s.cf" % (d, k), "rb").read() for k in "1234"]
    if name.startswith("adv_"):
        assert [len(x) for x in got] == [len(x) for x in want] and got == want, name
    else:
        util.assert_matches(got, want, name)


# ----------------------------------------------------------------------------- derived tables and the LF / resolve hooks
@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_tables_follow_the_geometry(name, monkeypatch):
    set_env(monkeypatch, {})
    base = index_base(name)
    ln, orate, fc, _, _ = header(base)
    assert (fc, orate) == GEOMETRIES[name]
    ix = capi().Index(base, 0)
    tb = ix.tables()
    k = kmer_k(fc, ln)
    assert (ix.info.ftab_chars, ix.info.off_rate) == (fc, orate)
    assert tb["ftab2_bytes"] == 16 << (2 * fc), tb
    assert tb["ftabk_chars"] == k and tb["ftabk_bytes"] == 16 << (2 * k) and tb["ftabd_chars"] == k + 3, tb
    if name in ("adv_t6o0", "adv_t1o2"):
        assert k == 8 > fc               # a K-mer table above ftabChars without a forcing knob
    ix.close()


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_lf_and_resolve_hooks_match_oracle(name):
    import ctypes as C
    m = capi()
    base = index_base(name)
    ln, orate, _, zoff, fchr = header(base)
    n_rows = ln + 1
    rng = np.random.default_rng(11)
    edges = [0, zoff, n_rows - 1] + list(fchr) + list(range(0, n_rows, 64)) + list(range(0, n_rows, 384)) + list(range(0, min(n_rows, 4096 << orate), 1 << orate))
    rows = np.array(sorted({r + d for r in edges for d in (-1, 0, 1) if 0 <= r + d < n_rows}
                           | set(range(400)) | set(range(n_rows - 400, n_rows))), dtype=np.uint64)
    rows = np.concatenate([rows, rng.integers(0, n_rows, size=20000).astype(np.uint64)])
    chars = rng.integers(0, 5, size=len(rows)).astype(np.uint8)        # 4 => the row's own BWT base
    ix = m.Index(base, 0)
    o = util.Oracle(base)
    o.lib.cfo_lf.restype = C.c_uint64
    o.lib.cfo_bwt_char.restype = C.c_int
    o.lib.cfo_resolve.restype = C.c_uint64
    got = m.test_lf(ix, rows, chars)
    gres = m.test_resolve(ix, rows)
    for i in range(len(rows)):
        r, c = C.c_uint64(int(rows[i])), int(chars[i])
        if c > 3:
            c = o.lib.cfo_bwt_char(C.c_void_p(o.h), r)
        assert int(got[i]) == o.lib.cfo_lf(C.c_void_p(o.h), r, C.c_int(c)), (name, i, int(rows[i]), c)
        assert int(gres[i]) == o.lib.cfo_resolve(C.c_void_p(o.h), r, None), (name, i, int(rows[i]))
    o.close(); ix.close()


# ----------------------------------------------------------------------------- records through the C ABI
def layouts(name):
    fc = GEOMETRIES[name][0]
    n_rows = header(index_base(name))[0] + 1
    return {"default": {}, "bitmap_only": {"CFB_FTABK": str(fc)}, "ftabk_plus2": {"CFB_FTABK": str(fc + 2)}, "no_bitmap": {"CFB_FTABD": "0"},
            "resolve_per_batch": {"CFB_RESOLVE_TABLE": "0"}, "partial_walk8": {"CFB_WALK8_ROWS": str(n_rows // 2)}, "keep_short": {"CFB_KEEP_SHORT": "1"}}


LAYOUTS = ["default", "bitmap_only", "ftabk_plus2", "no_bitmap", "resolve_per_batch", "partial_walk8", "keep_short"]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_records_match_oracle(name, layout, monkeypatch):
    set_env(monkeypatch, layouts(name)[layout])
    ix = capi().Index(index_base(name), 0)
    for rs, b in read_sets(name).items():
        for opt in sorted(OPTIONS):
            on, orec = oracle_records(name, opt, rs)
            gn, grec = gpu_records(ix, b, **OPTIONS[opt])
            try:
                assert_same(on, orec, gn, grec)
            except AssertionError as e:
                raise AssertionError("%s %s %s %s: %s" % (name, layout, rs, opt, e))
    ix.close()


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_counters_match_host_logic(name, monkeypatch):
    set_env(monkeypatch, {"CFB_COUNT": "1"})
    m = capi()
    base = index_base(name)
    h = util.HostLogic(base)
    ix = m.Index(base, 0)
    for rs, b in read_sets(name).items():
        _, _, hst = h.classify(b, util.make_oparams())
        ctx = m.Context(ix, m.make_params())
        ctx.classify(to_cbatch(b))
        c = ctx.counters()
        ctx.close()
        assert (c["partial_searches"], c["ftab_probes"], c["sides_search"], c["walk_steps"], c["rows_resolved"], c["ext_searches"]) \
            == (hst[1], hst[2], hst[3], hst[4], hst[5], hst[7]), (name, rs, c, hst)
    ix.close(); h.close()


def test_death_bitmap_gate_at_min_hitlen(monkeypatch):
    """-t 12: K = 12, so with --min-hitlen 15 every hit the bitmap can end (at most K + 2 bases) is shorter than min_hitlen and the
    bitmap is in use; at K = 13 it could end a 15-base hit, so it must be off.  The records are the oracle's either way."""
    m = capi()
    name = "syn_a_t12o5"
    b = read_sets(name)["se_1_300"]
    on, orec = oracle_records(name, "minhit15", "se_1_300")

    def run(env):
        set_env(monkeypatch, dict(env, CFB_COUNT="2"))
        ix = m.Index(index_base(name), 0)
        tb = ix.tables()
        ctx = m.Context(ix, m.make_params(min_hitlen=15))
        off, recs = ctx.classify(to_cbatch(b))
        req = ctx.requests()
        ctx.close(); ix.close()
        assert_same(on, orec, np.diff(off.astype(np.int64)).astype(np.uint32), recs)
        return tb, req
    tb, req = run({})
    assert tb["ftabk_chars"] == 12 and tb["ftabd_chars"] == 15, tb
    tb0, req0 = run({"CFB_FTABD": "0"})
    assert tb0["ftabk_bytes"] == 0, tb0
    assert req["rank16"] < req0["rank16"], (req, req0)
    tb13, _ = run({"CFB_FTABK": "13"})
    assert tb13["ftabk_chars"] == 13 and tb13["ftabd_chars"] == 16, tb13


@pytest.mark.parametrize("tables", ["default", "full"])
def test_cli_matches_reference_on_another_geometry(tables, adv_reads, tmp_path, monkeypatch):
    """centrifuge-class on the -t 6 -o 0 index, SE and PE FASTQ, with the CLI's lazy table set and with every table."""
    set_env(monkeypatch, {})
    if tables == "full":
        monkeypatch.setenv("CFB_FULL_TABLES", "1")
    else:
        monkeypatch.delenv("CFB_FULL_TABLES", raising=False)
    base = util.golden_index("adv_t6o0")
    reads = [(n, a) for n, a in util.parse_reads(adv_reads) if len(a) > 0 and n]
    f0, f1, f2 = str(tmp_path / "se.fq"), str(tmp_path / "p_1.fq"), str(tmp_path / "p_2.fq")
    util.synth.write_fastq(f0, reads)
    util.synth.write_fastq(f1, reads[:-1])
    util.synth.write_fastq(f2, [(n, revcomp(a)) for n, a in reads[1:]], qual=b"5")
    exe = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
    cases = {"se": ["-q", "-x", base, "-U", f0], "pe": ["-q", "-x", base, "-1", f1, "-2", f2]}
    wants = {tag: util.reference("gpu_geometry/cli_t6o0/" + tag, lambda: util.run_cli(util.REF_CLASS, args, str(tmp_path / "a.tsv"), str(tmp_path / "a.rep")))
             for tag, args in cases.items()}
    for tag, args in cases.items():
        want = wants[tag]
        util.assert_matches(util.run_cli(exe, args + ["--batch-units", "700"], str(tmp_path / "b.tsv"), str(tmp_path / "b.rep")), want, tables, tag)


# ----------------------------------------------------------------------------- the K-mer table's 24-bit width cap
# 67 Mbp of shuffled bases in 8 sequences, built at -t 1.  Loaded with CFB_FTABK=1 the K-mer table holds one entry per base whose
# width is that base's count: 2^24 - 2 is stored, 2^24 - 1 (= kFtabkWide) and above replay from the ftab, and a mask in place of
# the clamp would store 2^24 + 5 as a width of 5.
WIDE_COUNTS = (2 ** 24 - 2, 2 ** 24 - 1, 2 ** 24, 2 ** 24 + 5)


@functools.lru_cache(None)
def wide_genomes():
    rng = np.random.default_rng(2024)
    g = np.repeat(np.arange(4, dtype=np.uint8), WIDE_COUNTS)
    rng.shuffle(g)
    return np.array_split(g, 8)


@pytest.fixture(scope="module")
def wide_index():
    """(base, seconds the GPU builder took; None when cached)"""
    key = "width_cap_t1"
    d = os.path.join(util.CACHE, key)
    base = os.path.join(d, "idx")
    if os.path.exists(os.path.join(d, "done")):
        return base, None
    os.makedirs(d, exist_ok=True)
    seqs = wide_genomes()
    with open(os.path.join(d, "genomes.fa"), "wb") as f:
        for i, s in enumerate(seqs):
            a = util.synth.ACGT[s]
            full = len(a) // 80 * 80
            f.write(b">seq%d\n" % i + np.hstack([a[:full].reshape(-1, 80), np.full((full // 80, 1), 10, dtype=np.uint8)]).tobytes()
                    + a[full:].tobytes() + b"\n")
    conv, nodes, names = capi().write_synth_taxonomy(d, 2, 4, len(seqs[0]))
    t0 = time.time()
    util.build_cf([os.path.join(d, "genomes.fa")], conv, nodes, names, base, key, ftab_chars=1, off_rate=4)
    secs = time.time() - t0
    open(os.path.join(d, "done"), "w").close()
    return base, None if util.RECORD else secs


@pytest.mark.parametrize("bitmap", ["bitmap", "no_bitmap"])
def test_kmer_widths_at_the_24_bit_cap(bitmap, wide_index, monkeypatch):
    base, secs = wide_index
    if secs is not None:
        print("GPU builder, width-cap index (67 Mbp, -t 1): %.1f s" % secs)
    set_env(monkeypatch, {"CFB_FTABK": "1"} if bitmap == "bitmap" else {"CFB_FTABK": "1", "CFB_FTABD": "0"})
    ln, _, fc, _, fchr = header(base)
    assert fc == 1 and tuple(np.diff(fchr[:5])) == WIDE_COUNTS
    m = capi()
    ix = m.Index(base, 0)
    tb = ix.tables()
    if bitmap == "bitmap":
        assert tb["ftabk_chars"] == 1 and tb["ftabd_chars"] == 4, tb
    else:
        assert tb["ftabk_bytes"] == 0, tb
    b = util.Batch([a for _, a in util.synth.sample_reads(list(wide_genomes()), 2000, 100, seed=305, lens=(16, 200))])
    o = util.Oracle(base)
    for kw in ({}, dict(k=1), dict(min_hitlen=15)):
        on, orec, _ = o.classify(b, util.make_oparams(**kw))
        gn, grec = gpu_records(ix, b, **kw)
        assert_same(on, orec, gn, grec)
    o.close(); ix.close()
