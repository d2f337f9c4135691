"""GPU: walk8 jumps ranges of any width by their two end rows (DESIGN.md 3), in k_search_t and in search_strand_dev
(k_prep's list regeneration, k_search_long).

syn_a is strain-rich: after the K-mer jump the species of a genus share wide ranges.  The records must stay the oracle's with
walk8 covering all rows or only part of them (so that a range can have one end row covered and the other not), for single
reads, pairs and reads over 320 bases, with the default options, -k 1 and --min-hitlen 15."""
import pytest

import util
from test_gpu_parity import assert_same, gpu_classify, to_cbatch

pytestmark = pytest.mark.gpu

OPTIONS = {"default": {}, "k1": dict(k=1), "minhit15": dict(min_hitlen=15)}


def syn_a():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    return base, util.synth.make_genomes(5, 4, 60000, 7)


def batches(seqs):
    se = util.Batch([a for _, a in util.synth.sample_reads(seqs, 4000, 100, seed=91, lens=(60, 300))])
    prs = util.synth.sample_pairs(seqs, 2000, 150, seed=92)
    pe = util.Batch([x for _, x, _ in prs], [y for _, _, y in prs])
    long_se = util.Batch([a for _, a in util.synth.sample_reads(seqs, 1500, 321, seed=93, lens=(321, 800))])
    return {"se": se, "pe": pe, "long": long_se}


def variants(base):
    from centrifuge_b200 import capi as m
    ix = m.Index(base, 0)
    nrows = int(ix.info.len) + 1
    ix.close()
    return {"default": {}, "partial_walk8": {"CFB_WALK8_ROWS": str(nrows // 2)}}


@pytest.mark.parametrize("opt", sorted(OPTIONS))
def test_range_jumps_match_oracle(opt, monkeypatch):
    base, seqs = syn_a()
    bs = batches(seqs)
    o = util.Oracle(base)
    want = {k: o.classify(b, util.make_oparams(**OPTIONS[opt]))[:2] for k, b in bs.items()}
    o.close()
    for name, env in variants(base).items():
        monkeypatch.delenv("CFB_WALK8_ROWS", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        for k, b in bs.items():
            on, orec = want[k]
            gn, grec = gpu_classify(base, b, **OPTIONS[opt])
            assert_same(on, orec, gn, grec)


def test_wide_range_jumps_are_taken(monkeypatch):
    """CFB_COUNT=2: ranges of width >= 5 jump and the rank16 breakdown adds up."""
    from centrifuge_b200 import capi as m
    base, seqs = syn_a()
    b = batches(seqs)["se"]
    monkeypatch.setenv("CFB_COUNT", "2")
    ix = m.Index(base, 0)
    ctx = m.Context(ix, m.make_params())
    ctx.classify(to_cbatch(b))
    req, brk = ctx.requests(), ctx.request_breakdown()
    ctx.close(); ix.close()
    assert brk["rank16_w1"] + brk["rank16_w2_4"] + brk["rank16_w5"] == req["rank16"], (req, brk)
    assert brk["walk8_ok_w5"] > 0 and brk["walk8_ok_range"] >= brk["walk8_ok_w5"], brk
    assert brk["walk8_try_range"] >= brk["walk8_ok_range"] and brk["walk8_try_row"] >= brk["walk8_ok_row"] > 0, brk
