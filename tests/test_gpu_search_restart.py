"""GPU: the restart block of k_search_t -- the one copy of the hit store, the restart policy and the partial-search
prologue that every lane reaches at the end of a loop trip -- and the task hand-out that feeds it a read one trip after the
task was taken.  Records through the C ABI against the oracle for the reads that stress them: Ns inside the first 10-mer
(the prologue's loop over leading Ns), reads of Ns only, reads shorter than the 10-mer table's key, of exactly min_hitlen
bases, and of 128, 160 and 320 bases (the last base of the widest read each register window holds), batches whose task count
is not a multiple of a warp or of the hand-out chunk, and a batch smaller than one warp.  The table requests the counting
kernel reports for a fixed batch are pinned, so that a restructured loop still issues the same loads."""
import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, gpu_classify, to_cbatch

pytestmark = pytest.mark.gpu

N = ord("N")


def syn_a():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    return base, util.synth.make_genomes(5, 4, 60000, 7)


def reads_of(seqs, n, length, seed):
    return [a.copy() for _, a in util.synth.sample_reads(seqs, n, length, seed=seed, nrate=0.0)]


def check(base, batch, **kw):
    o = util.Oracle(base)
    on, orec, _ = o.classify(batch, util.make_oparams(**kw))
    o.close()
    gn, grec = gpu_classify(base, batch, **kw)
    assert_same(on, orec, gn, grec)
    return len(grec)


@pytest.mark.parametrize("length", [60, 150, 300])
def test_leading_ns_restart_the_prologue(length):
    """One to three Ns at every position of the first 10-mer, alone and in runs, and again right after the restart."""
    base, seqs = syn_a()
    rd = reads_of(seqs, 600, length, seed=300 + length)
    for i, r in enumerate(rd):
        p = i % 10
        r[len(r) - 1 - p] = N                      # strand 0 consumes the read from its end, strand 1 from its start
        r[p] = N
        if i % 3 == 1:
            r[p + 1] = N
        if i % 3 == 2:
            r[p + 11] = N                          # inside the 10-mer of the search that starts after the first N
            r[len(r) - 1 - p - 11] = N
    assert check(base, util.Batch(rd)) > 0


def test_reads_of_ns_only_and_short_reads():
    base, seqs = syn_a()
    rd = reads_of(seqs, 400, 100, seed=41)
    for i in range(0, 400, 5):
        rd[i] = np.full(20 + i % 90, N, dtype=np.uint8)
    for i in range(1, 400, 5):
        rd[i] = rd[i][: 1 + i % 9]                   # shorter than the 10-mer table's key
    for i in range(2, 400, 5):
        rd[i] = rd[i][:10 + i % 3]                   # the 10-mer and nothing, or little, after it
    check(base, util.Batch(rd))
    m2 = reads_of(seqs, 400, 100, seed=42)
    for i in range(3, 400, 7):
        m2[i] = m2[i][:0]                            # an empty mate next to a live one
    check(base, util.Batch(rd, m2))


@pytest.mark.parametrize("min_hitlen", [15, 22, 31])
def test_reads_of_exactly_min_hitlen(min_hitlen):
    base, seqs = syn_a()
    rd = [r[:min_hitlen + d] for d in (-1, 0, 1) for r in reads_of(seqs, 300, 60, seed=50 + min_hitlen + d)]
    check(base, util.Batch(rd), min_hitlen=min_hitlen)


@pytest.mark.parametrize("length", [96, 127, 128, 129, 159, 160, 161, 319, 320])
def test_last_base_of_every_register_window(length):
    """Reads that end on, before and after a 32-base word of the register window, at every window width."""
    base, seqs = syn_a()
    rd = reads_of(seqs, 700, length, seed=length)
    for i in range(0, len(rd), 9):
        rd[i][31 + 32 * (i % (length // 32))] = N    # an N on a word's last base
    assert check(base, util.Batch(rd)) > 0


@pytest.mark.parametrize("n", [1, 5, 31, 33, 257, 1000, 4099])
def test_task_counts_off_the_warp_and_the_chunk(n):
    base, seqs = syn_a()
    rd = reads_of(seqs, n, 100, seed=n)
    check(base, util.Batch(rd))
    if n > 1:
        m2 = reads_of(seqs, n, 100, seed=n + 1)
        m2[n // 2] = np.full(100, N, dtype=np.uint8)     # a filtered mate in the middle of the pool
        check(base, util.Batch(rd, m2))


REQUEST_BATCH = dict(n=6000, length=100, seed=2024, lens=(30, 300))
# counted at the commit before the restart block was merged into one copy
REQUESTS = ({"rank16": 105790, "ftab2": 55467, "ftabk": 105627, "walk8": 142605, "ftabd": 0},
            {"rank16_w1": 33052, "rank16_w2_4": 67084, "rank16_w5": 5654, "walk8_try_row": 64897, "walk8_ok_row": 59485,
             "walk8_try_range": 42664, "walk8_ok_range": 24671, "walk8_ok_w5": 70})


def request_batch(seqs):
    a = REQUEST_BATCH
    return util.Batch([r for _, r in util.synth.sample_reads(seqs, a["n"], a["length"], seed=a["seed"], lens=a["lens"])])


def count_requests(base, batch):
    from centrifuge_b200 import capi as m
    ix = m.Index(base, 0)
    ctx = m.Context(ix, m.make_params())
    ctx.classify(to_cbatch(batch))
    req, brk = ctx.requests(), ctx.request_breakdown()
    ctx.close(); ix.close()
    return req, brk


def test_table_requests_are_unchanged(monkeypatch):
    base, seqs = syn_a()
    monkeypatch.setenv("CFB_COUNT", "2")
    req, brk = count_requests(base, request_batch(seqs))
    assert (req, brk) == REQUESTS
