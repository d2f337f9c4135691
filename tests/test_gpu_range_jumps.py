"""GPU: walk8 jumps ranges of any width by their two end rows (DESIGN.md 3), in k_search_t and in search_strand_dev
(k_prep's list regeneration, k_search_long).

syn_a is strain-rich: after the K-mer jump the species of a genus share wide ranges.  The records must stay the oracle's with
the jump width capped (CFB_JUMP_W) or not, with walk8 covering only part of the rows (so that a range can have one end row
covered and the other not), for single reads, pairs and reads over 320 bases, with the default options, -k 1 and
--min-hitlen 15."""
import numpy as np
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
    return {"default": {}, "w1": {"CFB_JUMP_W": "1"}, "w4": {"CFB_JUMP_W": "4"},
            "partial_walk8": {"CFB_WALK8_ROWS": str(nrows // 2)}}


@pytest.mark.parametrize("opt", sorted(OPTIONS))
def test_range_jumps_match_oracle(opt, monkeypatch):
    base, seqs = syn_a()
    bs = batches(seqs)
    o = util.Oracle(base)
    want = {k: o.classify(b, util.make_oparams(**OPTIONS[opt]))[:2] for k, b in bs.items()}
    o.close()
    for name, env in variants(base).items():
        for k in ("CFB_JUMP_W", "CFB_WALK8_ROWS"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        for k, b in bs.items():
            on, orec = want[k]
            gn, grec = gpu_classify(base, b, **OPTIONS[opt])
            assert_same(on, orec, gn, grec)


def counted(base, b):
    from centrifuge_b200 import capi as m
    ix = m.Index(base, 0)
    ctx = m.Context(ix, m.make_params())
    off, recs = ctx.classify(to_cbatch(b))
    req, brk = ctx.requests(), ctx.request_breakdown()
    ctx.close(); ix.close()
    return off, recs, req, brk


def test_wide_range_jumps_are_taken_and_save_requests(monkeypatch):
    """CFB_COUNT=2: ranges of width >= 5 jump, the rank16 breakdown adds up, and the jump-width cap changes no record."""
    base, seqs = syn_a()
    b = batches(seqs)["se"]
    monkeypatch.setenv("CFB_COUNT", "2")
    off, recs, req, brk = counted(base, b)
    assert brk["rank16_w1"] + brk["rank16_w2_4"] + brk["rank16_w5"] == req["rank16"], (req, brk)
    assert brk["walk8_ok_w5"] > 0 and brk["walk8_ok_range"] >= brk["walk8_ok_w5"], brk
    assert brk["walk8_try_range"] >= brk["walk8_ok_range"] and brk["walk8_try_row"] >= brk["walk8_ok_row"] > 0, brk
    monkeypatch.setenv("CFB_JUMP_W", "4")
    off4, recs4, req4, brk4 = counted(base, b)
    assert brk4["walk8_ok_w5"] == 0, brk4
    assert np.array_equal(off, off4) and np.array_equal(recs, recs4)
    monkeypatch.setenv("CFB_JUMP_W", "1")
    _, _, _, brk1 = counted(base, b)
    assert brk1["walk8_try_range"] == 0 and brk1["walk8_try_row"] > 0, brk1
