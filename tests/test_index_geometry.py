"""CPU checks on indexes built with other -t/--ftabchars and -o/--offrate values than the default (10, 4).

The output depends on ftabChars (it sets where each partial search starts), and offRate sets how rows resolve, so the
default-geometry tests do not cover these indexes.  Per committed build of the adv genomes (tests/golden/adv_t<T>o<O>.*):
  * the oracle's file driver against the unmodified reference binary, TSV and report (by their recorded digest);
  * the product's per-thread logic (cf_logic.h compiled for the host) against the oracle, record by record, on the adv
    reads and on the random read sets of test_classify_fuzz, plus reads around ftabChars long;
  * the host-only loader reports the geometry."""
import random

import numpy as np
import pytest

import util
from test_classify_fuzz import make_reads
from util_fuzz import clean_reads

GEOMETRIES = {"adv_t6o0": (6, 0), "adv_t1o2": (1, 2), "adv_t8o7": (8, 7)}
CLI_CASES = {"default": [], "k1": ["-k", "1"], "k50": ["-k", "50"], "minhit15": ["--min-hitlen", "15"],
             "family": ["--classification-rank", "family"]}
API_OPTS = [dict(), dict(k=1), dict(k=50), dict(min_hitlen=15), dict(rank_slot=3), dict(traverse=False)]


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_oracle_cli_matches_reference(name, adv_reads, tmp_path):
    util.ensure_oracle()
    base = util.golden_index(name)
    for case, opts in sorted(CLI_CASES.items()):
        args = ["-f", "-x", base, "-U", adv_reads] + opts
        want = util.reference("geometry/%s/%s" % (name, case), lambda: util.run_cli(util.REF_CLASS, args, str(tmp_path / "r.tsv"), str(tmp_path / "r.rep")))
        util.assert_matches(util.run_cli(util.ORACLE_BIN, args, str(tmp_path / "o.tsv"), str(tmp_path / "o.rep")), want, name, case)
    # pairs: mate 2 of unit i is the reverse complement of read i + 1, so both strands of both mates hit
    reads = [(n, s) for n, s in clean_reads()][:1200]
    comp = bytes.maketrans(b"ACGTN", b"TGCAN")
    with open(tmp_path / "p1.fa", "wb") as f:
        f.write(b"".join(b">" + n + b"\n" + s + b"\n" for n, s in reads[:-1]))
    with open(tmp_path / "p2.fa", "wb") as f:
        f.write(b"".join(b">" + n + b"\n" + s[::-1].translate(comp) + b"\n" for n, s in reads[1:]))
    args = ["-f", "-x", base, "-1", str(tmp_path / "p1.fa"), "-2", str(tmp_path / "p2.fa")]
    want = util.reference("geometry/%s/paired" % name, lambda: util.run_cli(util.REF_CLASS, args, str(tmp_path / "r.tsv"), str(tmp_path / "r.rep")))
    util.assert_matches(util.run_cli(util.ORACLE_BIN, args, str(tmp_path / "o.tsv"), str(tmp_path / "o.rep")), want, name, "paired")


def short_reads(rng, reads, fc):
    """Reads of 0 .. ftabChars + 2 bases, from the genomes and random: the ftab lookup needs ftabChars of them."""
    out = []
    for L in range(0, fc + 3):
        for _ in range(3):
            a = rng.choice(reads)[1]
            out.append(a[:L])
        out.append(bytes(rng.choice(b"ACGT") for _ in range(L)))
    return out


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_product_logic_matches_oracle(name, adv_reads):
    util.ensure_oracle()
    base = util.golden_index(name)
    fc = GEOMETRIES[name][0]
    reads = clean_reads()
    o, h = util.Oracle(base), util.HostLogic(base)
    arr = lambda s: np.frombuffer(s, dtype=np.uint8)
    adv = util.Batch([a for _, a in util.parse_reads(adv_reads)])
    for kw in API_OPTS:
        p = util.make_oparams(**kw)
        on, orec, _ = o.classify(adv, p)
        hn, hrec, _ = h.classify(adv, p)
        assert np.array_equal(on, hn) and np.array_equal(orec, hrec), (name, kw)
    for case in range(60):
        rng = random.Random(50000 + case)
        rs = [s for _, s in make_reads(rng, reads)] + short_reads(rng, reads, fc)
        kw, paired = rng.choice(API_OPTS), rng.random() < 0.4
        if paired:
            rs2 = [s for _, s in make_reads(rng, reads)] + short_reads(rng, reads, fc)
            n = min(len(rs), len(rs2))
            bt = util.Batch([arr(s) for s in rs[:n]], [arr(s) for s in rs2[:n]])
        else:
            bt = util.Batch([arr(s) for s in rs])
        p = util.make_oparams(**kw)
        on, orec, _ = o.classify(bt, p)
        hn, hrec, _ = h.classify(bt, p)
        assert np.array_equal(on, hn) and np.array_equal(orec, hrec), (name, case, kw, paired)
    o.close(); h.close()


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_host_only_load_reports_the_geometry(name):
    from centrifuge_b200 import capi
    ix = capi.Index(util.golden_index(name), device=-1)
    fc, orate = GEOMETRIES[name]
    assert (ix.info.ftab_chars, ix.info.off_rate, ix.info.sample_bytes) == (fc, orate, 2)
    assert ix.info.line_rate == 7 and ix.info.len == 400200 and ix.info.n_seqs == 20
    ix.close()
