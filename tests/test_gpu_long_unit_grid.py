"""GPU: long units (a mate longer than 60 000 bases) across the -k / --min-hitlen grid, on the repeat-rich adv indexes at every
ftabChars / offRate geometry and on every device layout, against the oracle record by record.

Long units run their own kernels (k_long_seg, k_long_join, k_long_post, k_long_prep, k_long_score) on segments of 4 096 search
positions.  The reads (util_long.py) cross the tandem repeat, the A and T runs, the dispersed repeat and sequence 0 into its own
reverse complement; they are cut at 60 000 and 60 001 bases and at 4 096 k - 1, 4 096 k and 4 096 k + 1 bases, and carry Ns on
the last and first bases of segments, inside the first K-mer after a boundary and in a run across one.  Units are single reads,
long twins, long mates with short, empty or N-filtered partners, among short units at the per-unit stages' warp boundaries."""
import concurrent.futures
import functools
import os
import re
import subprocess

import numpy as np
import pytest

import util
import util_long as L
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu

INDEXES = ["adv", "adv_t1o2", "adv_t6o0", "adv_t8o7"]
OPTIONS = [(("k", k), ("min_hitlen", m)) for k in (1, 2, 5) for m in (15, 16, 17, 18, 21, 22, 23, 30)] \
    + [(("k", 1), ("min_hitlen", 15), ("rank_slot", 2)), (("k", 2), ("host", (100, 1005))), (("excl", (101,)),), (("traverse", False),)]
# the search tables change with the layout, the scoring stage does not: the whole grid on the default and compact layouts, the
# options that move the search (-k 1 and 5 at --min-hitlen 15, 17, 22 and 30) and the scoring points on the others
SEARCH_OPTIONS = [o for o in OPTIONS if o[-1][0] != "min_hitlen" or (o[0][1] in (1, 5) and o[1][1] in (15, 17, 22, 30))]
LAYOUTS = {"default": {}, "kmer_at_ftab": {"CFB_FTABK": "FC"}, "no_bitmap": {"CFB_FTABD": "0"}, "half_walk8": {"CFB_WALK8_ROWS": "HALF"},
           "resolve_per_batch": {"CFB_RESOLVE_TABLE": "0"}, "compact": {"CFB_RANK16": "0"}}
FULL_GRID = ("default", "compact")
KNOBS = ("CFB_RANK16", "CFB_FTABK", "CFB_FTABD", "CFB_RESOLVE_TABLE", "CFB_WALK8", "CFB_WALK8_ROWS", "CFB_KEEP_SHORT", "CFB_COUNT",
         "CFB_HBM_HEADROOM_GB", "CFB_REGEN_SLOTS", "CFB_REGEN_STATS", "CFB_ROWS_CAP")


def capi():
    from centrifuge_b200 import capi as m
    return m


def set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@functools.lru_cache(None)
def read_sets(name):
    """{set: (batch, long units in it)} for the index's K-mer table K"""
    k = L.kmer_k(name)
    se, _ = L.single_set(k)
    m1, m2 = L.pair_set(k)
    return {"se": (util.Batch(se), L.long_units_of(se)), "pe": (util.Batch(m1, m2), L.long_units_of(m1, m2))}


@functools.lru_cache(None)
def oracle_records(name, rs, opt):
    o = util.Oracle(util.golden_index(name))
    on, orec, _ = o.classify(read_sets(name)[rs][0], util.make_oparams(**dict(opt)))
    o.close()
    return on, orec


def prefetch_oracle(name):
    """every (read set, option) of the index through the oracle, on all CPUs (the oracle runs outside the GIL)"""
    keys = [(name, rs, opt) for rs in read_sets(name) for opt in OPTIONS]
    oracle_records(*keys[0])
    with concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(lambda a: oracle_records(*a), keys[1:]))


def classify(ctx, b):
    off, recs = ctx.classify(to_cbatch(b))
    return np.diff(off.astype(np.int64)).astype(np.uint32), recs


def open_layout(name, layout, monkeypatch):
    m = capi()
    base = util.golden_index(name)
    set_env(monkeypatch, {})
    ix = m.Index(base, 0)
    fc, rows, tb = ix.info.ftab_chars, ix.info.len + 1, ix.tables()
    ix.close()
    assert fc == L.FTAB_CHARS[name] and tb["ftabk_chars"] == L.kmer_k(name), tb
    set_env(monkeypatch, {k: v.replace("FC", str(fc)).replace("HALF", str(rows // 2)) for k, v in LAYOUTS[layout].items()})
    ix = m.Index(base, 0)
    tb = ix.tables()
    if layout == "compact":
        assert tb["rank16_bytes"] == 0, tb
    elif layout == "no_bitmap":
        assert tb["ftabd_chars"] == 0, tb
    else:
        assert tb["rank16_bytes"] > 0 and tb["ftabd_chars"] == tb["ftabk_chars"] + 3, tb
        if layout == "kmer_at_ftab":
            assert tb["ftabk_chars"] == fc, tb
    return ix


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("name", INDEXES)
def test_long_unit_grid_matches_oracle(name, layout, monkeypatch):
    prefetch_oracle(name)
    m = capi()
    ix = open_layout(name, layout, monkeypatch)
    sets = read_sets(name)
    bad = []
    try:
        for opt in OPTIONS if layout in FULL_GRID else SEARCH_OPTIONS:
            ctx = m.Context(ix, m.make_params(**dict(opt)))
            for rs, (b, n_long) in sets.items():
                before = ctx.long_stats()["units"]
                gn, grec = classify(ctx, b)
                got_long = ctx.long_stats()["units"] - before
                try:
                    assert got_long == n_long, "%d units took the long path, %d have a mate over %d bases" % (got_long, n_long, L.LONG)
                    assert_same(*oracle_records(name, rs, opt), gn, grec)
                except AssertionError as e:
                    bad.append("%s %s: %s" % (rs, dict(opt), e))
            ctx.close()
    finally:
        ix.close()
    assert not bad, "%s %s: %d cases differ from the oracle:\n%s" % (name, layout, len(bad), "\n".join(bad[:20]))


@pytest.mark.parametrize("name", INDEXES)
def test_threshold_takes_the_path_its_length_implies(name, monkeypatch):
    """60 000 bases: the short path (k_search_long); 60 001: the segmented path.  Same bases, records the oracle's."""
    set_env(monkeypatch, {})
    m = capi()
    lr = L.long_reads(L.kmer_k(name))
    ix = m.Index(util.golden_index(name), 0)
    o = util.Oracle(util.golden_index(name))
    shorts = L.short_reads(40, 91)
    for cut, want in (("cut60000", 0), ("cut60001", 1)):
        for b in (util.Batch(L.place([lr[cut]], shorts, [32])), util.Batch(L.place([lr[cut]], shorts, [5]), L.place([lr["cut60000"]], shorts, [5]))):
            for opt in ({}, dict(k=1, min_hitlen=15)):
                ctx = m.Context(ix, m.make_params(**opt))
                gn, grec = classify(ctx, b)
                assert ctx.long_stats()["units"] == want, (name, cut, ctx.long_stats())
                ctx.close()
                on, orec, _ = o.classify(b, util.make_oparams(**opt))
                assert_same(on, orec, gn, grec)
    o.close(); ix.close()


def unit_records(n, recs, i):
    off = np.concatenate([[0], np.cumsum(n.astype(np.int64))])
    return recs[off[i]:off[i + 1]]


@pytest.mark.parametrize("name", INDEXES)
def test_long_twins_reach_twin_removal(name, monkeypatch):
    """Pairs whose long mate 2 is mate 1's reverse complement against the same pairs with mate 2 replaced: both the oracle's,
    and the twins' records are not those of the replaced pairs."""
    set_env(monkeypatch, {})
    m = capi()
    k = L.kmer_k(name)
    twins = L.pair_units(k)
    repl = dict(twins, **L.replaced_twins(k))
    ix = m.Index(util.golden_index(name), 0)
    o = util.Oracle(util.golden_index(name))
    for opt in ({}, dict(k=1, min_hitlen=15)):
        got = []
        for units in (twins, repl):
            b = util.Batch(*L.pair_batch_of(units))
            ctx = m.Context(ix, m.make_params(**opt))
            gn, grec = classify(ctx, b)
            ctx.close()
            on, orec, _ = o.classify(b, util.make_oparams(**opt))
            assert_same(on, orec, gn, grec)
            got.append((gn, grec))
        for shape in ("twins_repeats", "twins_s0_s1"):
            i = L.PE_AT[L.PE_SHAPES.index(shape)]
            a, r = unit_records(*got[0], i), unit_records(*got[1], i)
            assert len(a) and not np.array_equal(a, r), (name, opt, shape)
    o.close(); ix.close()


@pytest.mark.parametrize("name", ["adv", "adv_t8o7"])
def test_row_buffer_overflow_reruns_the_tail(name, monkeypatch):
    """CFB_ROWS_CAP=64: the long units' rows overflow the row buffer, k_long_score returns early and the host runs the row stage
    again (k_long_prep<true> re-emits the rows).  A batch of three long units fits the default buffer; under the cap it is
    launched again, and the records are the oracle's."""
    m = capi()
    lr = L.long_reads(L.kmer_k(name))
    only_long = util.Batch([lr["repeats"], lr["s0_s1"], lr["chimera"]])
    sets = {"only_long": only_long, "se": read_sets(name)["se"][0], "pe": read_sets(name)["pe"][0]}
    o = util.Oracle(util.golden_index(name))
    launches = {}
    for cap in (None, "64"):
        set_env(monkeypatch, {"CFB_ROWS_CAP": cap} if cap else {})
        ix = m.Index(util.golden_index(name), 0)
        for rs, b in sets.items():
            for opt in ({}, dict(k=1, min_hitlen=15)):
                ctx = m.Context(ix, m.make_params(**opt))
                gn, grec = classify(ctx, b)
                launches[cap, rs, tuple(opt)] = ctx.launches()
                ctx.close()
                on, orec, _ = o.classify(b, util.make_oparams(**opt))
                assert_same(on, orec, gn, grec)
        ix.close()
    o.close()
    for (cap, rs, opt), n in launches.items():
        if cap and rs == "only_long":
            assert n > launches[None, rs, opt], (name, rs, opt, launches)


@pytest.mark.parametrize("name", INDEXES)
def test_counters_match_host_logic(name, monkeypatch):
    """CFB_COUNT=1: the long units' strands are searched by the scalar join; every count equals the host logic's"""
    set_env(monkeypatch, {"CFB_COUNT": "1"})
    m = capi()
    base = util.golden_index(name)
    h = util.HostLogic(base)
    ix = m.Index(base, 0)
    for rs, (b, _) in read_sets(name).items():
        for opt in ({}, dict(k=1, min_hitlen=15)):
            _, _, hst = h.classify(b, util.make_oparams(**opt))
            ctx = m.Context(ix, m.make_params(**opt))
            classify(ctx, b)
            c = ctx.counters()
            ctx.close()
            assert (c["partial_searches"], c["ftab_probes"], c["sides_search"], c["walk_steps"], c["rows_resolved"], c["ext_searches"]) \
                == (hst[1], hst[2], hst[3], hst[4], hst[5], hst[7]), (name, rs, opt, c, hst)
    ix.close(); h.close()


@pytest.mark.parametrize("name", ["adv", "adv_t6o0"])
def test_packed_and_resident_windows(name, monkeypatch):
    """The packed form and resident windows cut between two long units give the byte form's records."""
    set_env(monkeypatch, {})
    m = capi()
    ix = m.Index(util.golden_index(name), 0)
    for opt in ({}, dict(k=1, min_hitlen=15)):
        ctx = m.Context(ix, m.make_params(**opt))
        for rs, (b, _) in read_sets(name).items():
            cb = to_cbatch(b)
            off0, rec0 = ctx.classify(cb)
            off0 = off0.astype(np.int64)
            words, npos = m.pack_batch(cb)
            len2, flags = (b.len2, b.flags & 3) if b.paired else (None, b.flags & 1)
            ctx.submit_packed(1, m.make_batch_packed(words, b.len1, len2, npos, flags.astype(np.uint8)))
            off1, rec1 = ctx.wait(1)
            assert np.array_equal(off0, off1.astype(np.int64)) and np.array_equal(rec0, rec1), (name, rs)
            at = L.SE_AT if rs == "se" else L.PE_AT
            cuts = [c for c in at if c - 1 in at]              # between two long units
            assert cuts
            d = ctx.upload(cb)
            for c in cuts:
                for lo, hi in ((0, c), (c, b.n), (c - 1, c + 1)):
                    ctx.classify_resident(d, lo, hi - lo)
                    off2, rec2 = ctx.resident_result()
                    assert np.array_equal(rec2, rec0[off0[lo]:off0[hi]]), (name, rs, lo, hi)
                    assert np.array_equal(off2.astype(np.int64), off0[lo:hi + 1] - off0[lo]), (name, rs, lo, hi)
            m.lib().cfb_dbatch_free(ctx.h, d)
        ctx.close()
    ix.close()


# ------------------------------------------------------------------------------ centrifuge-class on files with long units
EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")


@pytest.fixture(scope="module")
def cli_cases(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("longunits"))
    return {c[0]: c for c in L.cli_cases(d, util.golden_index("adv"))}


def run_cli(args, tmp, tag):
    tsv, rep = str(tmp / (tag + ".tsv")), str(tmp / (tag + ".rep"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                       env=dict(os.environ, CFB_TEXT_STATS="1"))
    err = p.stderr.decode()
    assert p.returncode == 0, err
    t = re.search(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units", err)
    lu = re.search(r"long units: (\d+) \((\d+) bases\)", err)
    st = dict(text=int(t.group(1)), fallbacks=int(t.group(3)), host=int(t.group(4)), long=int(lu.group(1)))
    return tuple(open(x, "rb").read() for x in (tsv, rep)), st


@pytest.mark.parametrize("case", [c[0] for c in L.cli_cases()])
def test_cli_long_units_match_reference(cli_cases, case, tmp_path, monkeypatch):
    set_env(monkeypatch, {})
    key, args, n_units, n_long = cli_cases[case]
    want = L.ref_digest(key, args, tmp_path)
    got, st = run_cli(args, tmp_path, "text")
    util.assert_matches(got, want, case)
    assert st["fallbacks"] == 0 and st["host"] == 0 and st["text"] == n_units and st["long"] == n_long, (case, st, n_long)
    got_h, st_h = run_cli(args + ["--host-parse"], tmp_path, "host")
    assert got_h == got and st_h["host"] == n_units and st_h["long"] == n_long, (case, st_h)
