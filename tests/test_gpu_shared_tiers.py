"""k_score keeps a warp's hit maps in shared memory when the warp's span of rows fits its CTA's pool, and in the global
scratch otherwise.  One batch that needs both tiers must give the oracle's records."""
import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, gpu_classify

pytestmark = pytest.mark.gpu

SCORE_POOL = 128      # kScorePool: rows per CTA of k_score (cfb200.cu)
WARPS_PER_CTA = 4     # kScoreThreads / 32


def rows_per_warp(base, b, reads):
    """SA rows each warp of 32 consecutive units resolves, counted by the host twin of the per-unit logic."""
    h = util.HostLogic(base)
    out = []
    for s in range(0, b.n, 32):
        _, _, ctr = h.classify(util.Batch([a for _, a in reads[s:s + 32]]), util.make_oparams(), counters=True)
        out.append(ctr[5])
    h.close()
    return np.array(out, dtype=np.int64)


def test_shared_and_global_hit_maps_in_one_batch():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    seqs = util.synth.make_genomes(5, 4, 60000, 7)
    # CTAs of mostly random reads resolve few rows and keep their maps in shared memory; CTAs of long reads from the
    # strains of a species resolve many rows per unit and overflow the pool
    reads = util.synth.sample_reads(seqs, 1024, 100, seed=5, random_frac=0.95) + util.synth.sample_reads(seqs, 2048, 100, seed=6, lens=(150, 400))
    b = util.Batch([a for _, a in reads])
    w = rows_per_warp(base, b, reads)
    cta = np.add.reduceat(w, np.arange(0, len(w), WARPS_PER_CTA))
    assert (w > SCORE_POOL).any(), "no warp needs the global scratch"
    assert ((cta > 0) & (cta <= SCORE_POOL)).any(), "no CTA keeps all its warps' hit maps in shared memory"
    o = util.Oracle(base)
    on, orec, _ = o.classify(b, util.make_oparams())
    o.close()
    gn, grec = gpu_classify(base, b)
    assert_same(on, orec, gn, grec)
