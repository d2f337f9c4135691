"""The scoring stage behind the search (k_score, the record scan, k_compact, k_fold_counts) against the oracle, on the cases its
code paths split on: -k 1 and -k 5, the exclude and
host sets, --classification-rank, --no-traverse, paired units, warps whose hit maps do not fit the shared pool, and an index
with more than 65 535 sequences.  Every case compares the records with the oracle's.  The counting instantiation of k_score
(CFB_COUNT=2) reports which paths a batch took; the cases whose path this small index reaches only on some inputs check that
they reached it: -k 1 the tree reduction over several rank rounds, the long reads the global scratch.  -k 5 runs no tree
reduction here (no unit has more than five tied sequences on this index); the bench index, with ten species per genus, has them."""
import numpy as np
import pytest

import util
import util_wide
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu


def capi():
    from centrifuge_b200 import capi as m
    return m


def classify_with_stats(base, b, monkeypatch, **kw):
    """records of the batch, and k_score's statistics of the same batch from a counting context"""
    m = capi()
    ix = m.Index(base, 0)
    ctx = m.Context(ix, m.make_params(**kw))
    off, recs = ctx.classify(to_cbatch(b))
    ctx.close()
    monkeypatch.setenv("CFB_COUNT", "2")
    cctx = m.Context(ix, m.make_params(**kw))
    off2, recs2 = cctx.classify(to_cbatch(b))
    st = cctx.score_stats()
    cctx.close()
    monkeypatch.delenv("CFB_COUNT")
    ix.close()
    assert np.array_equal(off, off2) and np.array_equal(recs, recs2), "the counting instantiation of k_score gives other records"
    return np.diff(off.astype(np.int64)).astype(np.uint32), recs, st


def check(base, b, monkeypatch, **kw):
    o = util.Oracle(base)
    on, orec, _ = o.classify(b, util.make_oparams(**kw))
    o.close()
    gn, grec, st = classify_with_stats(base, b, monkeypatch, **kw)
    assert_same(on, orec, gn, grec)
    return st


def syn_a():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    return base, util.synth.make_genomes(5, 4, 60000, 7)


CASES = {
    "k1": dict(k=1), "k5": dict(k=5), "k2_host": dict(k=2, host=(100, 1005)), "excl": dict(excl=(10,)),
    "family": dict(rank_slot=3), "genus_k1": dict(rank_slot=2, k=1), "notraverse": dict(traverse=False),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_single_end_cases_match_oracle(case, monkeypatch):
    base, seqs = syn_a()
    b = util.Batch([a for _, a in util.synth.sample_reads(seqs, 6000, 100, seed=501, lens=(40, 250))])
    st = check(base, b, monkeypatch, **CASES[case])
    assert st["units"] > 0 and st["distinct_ids"] >= st["units"]
    if case == "k1":          # strain-rich genera: more than one tied sequence, reduced over several rank rounds
        assert st["reduce_units"] > 0 and st["reduce_rounds"] > st["reduce_units"], st


def test_paired_units_match_oracle(monkeypatch):
    base, seqs = syn_a()
    prs = util.synth.sample_pairs(seqs, 4000, 150, seed=502)
    m1 = [x for _, x, _ in prs]; m2 = [y for _, _, y in prs]
    for i in range(0, len(m2), 9):
        m2[i] = np.full(len(m2[i]), ord("N"), dtype=np.uint8)
    bp = util.Batch(m1, m2)
    for kw in ({}, dict(k=1)):
        st = check(base, bp, monkeypatch, **kw)
        assert st["units"] > 0


def test_warps_on_the_global_scratch_match_oracle(monkeypatch):
    """Long reads give units of many rows, so whole warps' hit maps do not fit the shared pool and live in global memory."""
    base, seqs = syn_a()
    b = util.Batch([a for _, a in util.synth.sample_reads(seqs, 3000, 600, seed=503, lens=(400, 900))])
    for kw in ({}, dict(k=1)):
        st = check(base, b, monkeypatch, **kw)
        assert st["warps_global"] > 0, st


def test_more_than_65535_sequences_match_oracle(monkeypatch):
    """u32 sequence ids: the per-context sequence table covers every id."""
    base, g = util_wide.wide_index()
    rng = np.random.default_rng(45)
    A = util.synth.ACGT
    b = util.Batch([A[g[int(rng.integers(60000, util_wide.N))][:100]].copy() for _ in range(3000)])     # high ids, past 65 535
    for kw in ({}, dict(k=1), dict(rank_slot=2, excl=(1003,))):
        st = check(base, b, monkeypatch, **kw)
        assert st["units"] > 0
