"""GPU: the -k / --min-hitlen grid of the host fast-path test (test_fast_path_rules_host.py) on the device, through the C ABI,
against the oracle record by record, on every device layout and with reads that select every search kernel.

The rank16 path stores hit lists with less in them than the exact search (hits the death bitmap ends have no SA range; with
--min-hitlen >= 22 only the long hits are stored) and restores what matters by rules that depend on -k, --min-hitlen, pairs and
the index geometry together; each option alone is tested elsewhere.  Layouts: the default tables, the K-mer table at K =
ftabChars (bitmap only), no bitmap, every hit stored, walk8 on half of the rows, and the compact rank layout.  Read lengths:
<= 128, 129-160, 161-320 bases (k_search_t with 4, 5 and 10 register words) and beyond 320 (k_search_long)."""
import functools
import lzma
import os
import re

import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu

INDEXES = ["example", "adv", "adv_t1o2", "adv_t6o0", "adv_t8o7"]
OPTIONS = [(("k", k), ("min_hitlen", m)) for k in (1, 2, 5) for m in (15, 16, 17, 18, 21, 22, 23, 30)] + [(("k", 1), ("min_hitlen", 15), ("rank_slot", 2))]
LAYOUTS = {"default": {}, "kmer_at_ftab": {"CFB_FTABK": "FC"}, "no_bitmap": {"CFB_FTABD": "0"}, "keep_short": {"CFB_KEEP_SHORT": "1"},
           "half_walk8": {"CFB_WALK8_ROWS": "HALF"}, "compact": {"CFB_RANK16": "0"}}
KNOBS = ("CFB_RANK16", "CFB_FTABK", "CFB_FTABD", "CFB_RESOLVE_TABLE", "CFB_WALK8", "CFB_WALK8_ROWS", "CFB_KEEP_SHORT", "CFB_COUNT",
         "CFB_HBM_HEADROOM_GB", "CFB_REGEN_SLOTS", "CFB_REGEN_STATS", "CFB_ROWS_CAP")
LENGTHS = {"r128": (1, 128), "r160": (129, 160), "r320": (161, 320), "r900": (321, 900)}


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
    if name == "example":
        return [a for _, a in util.parse_reads(os.path.join(util.GOLDEN, "example.reads.fa"))]
    fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
    if not os.path.exists(fa):
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa + ".tmp", "wb") as g:
            g.write(f.read())
        os.replace(fa + ".tmp", fa)
    return [a for _, a in util.parse_reads(fa)]


@functools.lru_cache(None)
def read_sets(name):
    """Per length class: SE reads, and pairs whose mate 2 is mate 1's reverse complement or another read of the class.  Reads
    are the index's own reads, cut to the class or joined (alternately reverse-complemented) up to it."""
    rs = reads_of(name)
    rng = np.random.default_rng(7 + len(name))
    sets = {}
    for cls, (lo, hi) in LENGTHS.items():
        n = 12 if name == "example" else (240 if hi <= 320 else 80)
        out, q = [], int(rng.integers(0, len(rs)))
        while len(out) < n:
            want = int(rng.integers(lo, hi + 1))
            parts, have = [], 0
            while have < want:
                x = rs[q % len(rs)]; q += 1
                parts.append(revcomp(x) if len(parts) % 2 else x); have += len(x)
            out.append(np.ascontiguousarray(np.concatenate(parts)[:want]))
        assert max(len(x) for x in out) > lo or lo == 1
        pairs = [(out[i], revcomp(out[i]) if i % 2 == 0 else out[(i * 7 + 3) % n]) for i in range(n)]
        sets[cls + "_se"] = util.Batch(out)
        sets[cls + "_pe"] = util.Batch([x for x, _ in pairs], [y for _, y in pairs])
    return sets


@functools.lru_cache(None)
def oracle_records(name, rs, opt):
    o = util.Oracle(util.golden_index(name))
    on, orec, _ = o.classify(read_sets(name)[rs], util.make_oparams(**dict(opt)))
    o.close()
    return on, orec


def gpu_records(ix, batches, opt):
    m = capi()
    ctx = m.Context(ix, m.make_params(**dict(opt)))
    out = {}
    for rs, b in batches.items():
        off, recs = ctx.classify(to_cbatch(b))
        out[rs] = (np.diff(off.astype(np.int64)).astype(np.uint32), recs)
    ctx.close()
    return out


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("name", INDEXES)
def test_option_grid_matches_oracle(name, layout, monkeypatch):
    m = capi()
    base = util.golden_index(name)
    set_env(monkeypatch, {})
    ix = m.Index(base, 0)
    fc, rows = ix.info.ftab_chars, ix.info.len + 1
    ix.close()
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
    sets = read_sets(name)
    bad = []
    try:
        for opt in OPTIONS:
            for rs, (gn, grec) in gpu_records(ix, sets, opt).items():
                on, orec = oracle_records(name, rs, opt)
                try:
                    assert_same(on, orec, gn, grec)
                except AssertionError as e:
                    bad.append("%s %s: %s" % (rs, dict(opt), e))
    finally:
        ix.close()
    assert not bad, "%s %s: %d cases differ from the oracle:\n%s" % (name, layout, len(bad), "\n".join(bad[:20]))


def test_regeneration_buffer_overflow(monkeypatch, capfd):
    """--min-hitlen 22 (only long hits stored, lists regenerated where both strands are in play) with a side buffer of two
    lists: k_prep overflows it, the host grows it and re-runs the batch; the records are still the oracle's."""
    m = capi()
    name = "adv_t1o2"
    set_env(monkeypatch, {"CFB_REGEN_SLOTS": "2", "CFB_REGEN_STATS": "1"})
    ix = m.Index(util.golden_index(name), 0)
    sets = {rs: b for rs, b in read_sets(name).items() if rs in ("r128_pe", "r160_pe", "r320_pe")}
    capfd.readouterr()
    try:
        for opt in ((("k", 1), ("min_hitlen", 22)), (("k", 5), ("min_hitlen", 23))):
            for rs, (gn, grec) in gpu_records(ix, sets, opt).items():
                assert_same(*oracle_records(name, rs, opt), gn, grec)
    finally:
        ix.close()
    err = capfd.readouterr().err
    got = [int(x) for x in re.findall(r"strand lists regenerated by k_prep: (\d+) of", err)]
    assert got and min(got) > 2, err
