"""GPU: a batch with a read over 320 bases, too long for k_search_t's register window, is searched by k_search_long on rank16.

The loader frees the file's sides once rank16 is built, whatever the index size, so the small fixture index here has the
device layout of a big one."""
import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, gpu_classify, to_cbatch

pytestmark = pytest.mark.gpu

OPTIONS = {"default": {}, "k1": dict(k=1), "minhit15": dict(min_hitlen=15)}


def syn_a():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    return base, util.synth.make_genomes(5, 4, 60000, 7)


def long_se(seqs, n=3000):
    return util.Batch([a for _, a in util.synth.sample_reads(seqs, n, 321, seed=41, lens=(321, 1000))])


def long_pairs(seqs):
    prs = util.synth.sample_pairs(seqs, 2000, 400, seed=42)
    m1 = [x for _, x, _ in prs]; m2 = [y for _, _, y in prs]
    for i in range(0, len(m2), 7):                          # filtered / very short mates
        m2[i] = np.full(len(m2[i]), ord("N"), dtype=np.uint8)
    for i in range(3, len(m1), 11):
        m1[i] = np.full(len(m1[i]), ord("N"), dtype=np.uint8)
    for i in range(5, len(m2), 13):
        m2[i] = m2[i][:1]
    return util.Batch(m1, m2)


def test_sides_are_freed_at_load():
    from centrifuge_b200 import capi as m
    base, _ = syn_a()
    ix = m.Index(base, 0)
    assert ix.tables()["sides_bytes"] == 0
    ix.close()


@pytest.mark.parametrize("opt", sorted(OPTIONS))
def test_long_reads_match_oracle(opt):
    base, seqs = syn_a()
    o = util.Oracle(base)
    for b in (long_se(seqs), long_pairs(seqs)):
        assert max(int(b.len1.max()), int(b.len2.max())) > 320
        on, orec, _ = o.classify(b, util.make_oparams(**OPTIONS[opt]))
        gn, grec = gpu_classify(base, b, **OPTIONS[opt])
        assert_same(on, orec, gn, grec)
    o.close()


def test_long_read_counters_match_host_logic(monkeypatch):
    """CFB_COUNT=1 on reads over 320 bases: the scalar search (search_strand_scalar, the host logic's own search) counts the
    reference's operations on the device, as it does for reads of every length."""
    monkeypatch.setenv("CFB_COUNT", "1")
    from centrifuge_b200 import capi as m
    base, seqs = syn_a()
    b = long_se(seqs, 1000)
    h = util.HostLogic(base)
    _, _, hst = h.classify(b, util.make_oparams())
    h.close()
    ix = m.Index(base, 0); ctx = m.Context(ix, m.make_params())
    ctx.classify(to_cbatch(b))
    c = ctx.counters()
    ctx.close(); ix.close()
    assert c["partial_searches"] == hst[1] and c["ftab_probes"] == hst[2] and c["sides_search"] == hst[3]
    assert c["walk_steps"] == hst[4] and c["rows_resolved"] == hst[5] and c["ext_searches"] == hst[7]


def test_packed_long_reads_match_byte_form():
    from centrifuge_b200 import capi as m
    base, seqs = syn_a()
    ix = m.Index(base, 0); ctx = m.Context(ix)
    for b in (long_se(seqs), long_pairs(seqs)):
        cb = to_cbatch(b)
        off0, rec0 = ctx.classify(cb)
        words, npos = m.pack_batch(cb)
        assert len(npos) > 0
        len2, flags = (b.len2, b.flags & 3) if b.paired else (None, b.flags & 1)
        ctx.submit_packed(1, m.make_batch_packed(words, b.len1, len2, npos, flags.astype(np.uint8)))
        off1, rec1 = ctx.wait(1)
        assert np.array_equal(off0, off1) and np.array_equal(rec0, rec1)
    ctx.close(); ix.close()
