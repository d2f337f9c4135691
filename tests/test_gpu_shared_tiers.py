"""k_score keeps a warp's hit maps in shared memory when the warp's span of rows fits its CTA's pool, and in the global
scratch otherwise.  One batch that needs both tiers must give the oracle's records; the counting instantiation of k_score
(CFB_COUNT=2) shows that it used both."""
import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, gpu_classify, to_cbatch

pytestmark = pytest.mark.gpu


def test_shared_and_global_hit_maps_in_one_batch(monkeypatch):
    from centrifuge_b200 import capi
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    seqs = util.synth.make_genomes(5, 4, 60000, 7)
    # CTAs of mostly random reads resolve few rows and keep their maps in shared memory; CTAs of long reads from the
    # strains of a species resolve many rows per unit and overflow the pool
    reads = util.synth.sample_reads(seqs, 1024, 100, seed=5, random_frac=0.95) + util.synth.sample_reads(seqs, 2048, 100, seed=6, lens=(150, 400))
    b = util.Batch([a for _, a in reads])
    o = util.Oracle(base)
    on, orec, _ = o.classify(b, util.make_oparams())
    o.close()
    assert_same(on, orec, *gpu_classify(base, b))
    monkeypatch.setenv("CFB_COUNT", "2")
    ix = capi.Index(base, 0)
    ctx = capi.Context(ix)
    off, grec = ctx.classify(to_cbatch(b))
    st = ctx.score_stats()
    ctx.close(); ix.close()
    assert 0 < st["warps_global"] < st["warps"], st
    assert_same(on, orec, np.diff(off.astype(np.int64)).astype(np.uint32), grec)
