"""GPU: the death bitmap rides in the K-mer jump table's 16-byte entries (DESIGN.md 3).

On an index too small for a K-mer table above ftabChars, the table is built at K = ftabChars for the bitmap alone.  The bitmap
must leave the records unchanged while it saves rank gathers, and it is read with the K-mer entry: no request of its own."""
import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu


def run(base, b):
    from centrifuge_b200 import capi as m
    ix = m.Index(base, 0)
    tb, fc = ix.tables(), ix.info.ftab_chars
    ctx = m.Context(ix)
    off, recs = ctx.classify(m.make_batch(b.bases, b.off1, b.len1, None, None, (b.flags & 1).astype(np.uint8)))
    req = ctx.requests()
    ctx.close(); ix.close()
    return tb, fc, off, recs, req


def test_small_index_gets_the_death_bitmap_in_a_kmer_table_at_ftab_chars(adv_base, adv_reads, monkeypatch):
    b = util.Batch([a for _, a in util.parse_reads(adv_reads)])
    monkeypatch.setenv("CFB_COUNT", "2")               # the kernel counts its own load requests per table
    tb, fc, off, recs, req = run(adv_base, b)
    assert tb["ftabk_chars"] == fc and tb["ftabk_bytes"] == 16 << (2 * fc), tb
    assert tb["ftabd_bytes"] == 0 and tb["ftabd_chars"] == fc + 3, tb
    monkeypatch.setenv("CFB_FTABD", "0")               # no bitmap wanted: no K-mer table at K = ftabChars either
    tb0, _, off0, recs0, req0 = run(adv_base, b)
    assert tb0["ftabk_bytes"] == 0 and tb0["ftabd_chars"] == 0, tb0
    assert np.array_equal(off, off0) and np.array_equal(recs, recs0)
    assert req["ftabd"] == 0 and req0["ftabd"] == 0
    assert req["ftabk"] > 0 and req0["ftabk"] == 0
    assert req["rank16"] < req0["rank16"], (req, req0)
