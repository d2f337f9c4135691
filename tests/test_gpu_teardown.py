"""Closing what the library creates gives back every byte of device memory.  For each owner (index, context, decoders, EM,
builder, measurement and test hooks) one warm-up cycle of create, use and close runs first: lazy module loading and local-memory
growth stay with the process.  Three more identical cycles must then leave the free device memory exactly where the warm-up left
it.  The context runs with small row and regeneration buffers (CFB_ROWS_CAP, CFB_REGEN_SLOTS) so that its grow-and-re-run paths
allocate too."""
import bz2
import gzip

import numpy as np
import pytest

import util
from test_gpu_compact_rank import capi, read_sets, reads_of
from test_gpu_parity import to_cbatch
from util_em import device_em, random_problem

pytestmark = pytest.mark.gpu

CFB_EDATA = -7


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def assert_cycles_return_memory(cycle):
    cycle()
    before = free_bytes()
    for i in range(3):
        cycle()
        after = free_bytes()
        assert after == before, "cycle %d kept %d bytes of device memory" % (i, before - after)


def fastq(reads):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, a.tobytes(), b"I" * len(a)) for i, a in enumerate(reads))


@pytest.mark.parametrize("rank16", [True, False])
def test_index(rank16, monkeypatch):
    m = capi()
    base = util.golden_index("adv")
    for k in ("CFB_RANK16", "CFB_HBM_HEADROOM_GB", "CFB_RESOLVE_TABLE", "CFB_WALK8", "CFB_FTABK", "CFB_FTABD"):
        monkeypatch.delenv(k, raising=False)
    if not rank16:
        monkeypatch.setenv("CFB_RANK16", "0")
    b = to_cbatch(util.Batch(reads_of("adv")[:200]))

    def cycle():
        ix = m.Index(base, 0)
        t = ix.tables()
        if rank16:
            assert t["rank16_bytes"] and t["ftabk_bytes"] and t["resolve_table_bytes"] and t["walk8_bytes"], t
        else:
            assert t["rank16_bytes"] == 0 and t["sides_bytes"], t
        ctx = m.Context(ix)
        ctx.classify(b)
        ctx.close()
        ix.close()
    assert_cycles_return_memory(cycle)


def test_context(monkeypatch):
    m = capi()
    monkeypatch.setenv("CFB_ROWS_CAP", "64")
    monkeypatch.setenv("CFB_REGEN_SLOTS", "1")
    ix = m.Index(util.golden_index("adv"), 0)
    sets = read_sets("adv")
    long_b, pe = sets["long_se"], sets["pe"]
    assert long_b.len1.max() > 60000
    cb_long, cb_pe = to_cbatch(long_b), to_cbatch(pe)
    words, npos = m.pack_batch(cb_pe)
    packed = m.make_batch_packed(words, pe.len1, pe.len2, npos, (pe.flags & 3).astype(np.uint8))
    rs = reads_of("adv")
    short_text = np.frombuffer(fastq(rs[:300]), dtype=np.uint8).copy()
    long_text = np.frombuffer(fastq(rs[:100] + [np.concatenate(rs[:700])[:61000]] + rs[100:200]), dtype=np.uint8).copy()

    def cycle():
        ctx = m.Context(ix)
        ctx.classify(cb_long)
        ctx.submit_packed(1, packed)
        ctx.wait(1)
        ctx.text_submit(2, short_text, None, 300)
        ctx.text_wait(2)
        ctx.text_submit(3, long_text, None, 201)
        ctx.text_wait(3)
        d = ctx.upload(cb_pe)
        ctx.classify_resident(d, 100, 300)
        ctx.resident_result()
        ctx.close()
    assert_cycles_return_memory(cycle)
    ix.close()


@pytest.mark.parametrize("kind", ["gzip", "bzip2"])
def test_decoders(kind):
    m = capi()
    data = fastq(reads_of("adv")[:5000])
    if kind == "gzip":
        comp, cls = gzip.compress(data), m.Gunzip
        bad = bytearray(comp); bad[-8] ^= 1                 # the member's CRC-32
    else:
        comp, cls = bz2.compress(data), m.Bunzip2
        bad = bytearray(comp); bad[10] ^= 1                 # the first block's CRC
    bad = bytes(bad)

    def cycle():
        g = cls(0)
        assert g.decompress(comp) == data
        g.close()
        g = cls(0)
        with pytest.raises(m.CfbError) as e:
            g.decompress(bad)
        assert e.value.code == CFB_EDATA, str(e.value)
        g.close()
    assert_cycles_return_memory(cycle)


def test_em():
    problem = random_problem(3, 300, 3000)
    assert_cycles_return_memory(lambda: device_em(*problem))


def test_build_index(tmp_path):
    m = capi()
    d = str(tmp_path)
    conv, nodes, names = m.write_synth_taxonomy(d, 4, 5, 30000)
    runs = iter(range(4))

    def cycle():
        m.build_index(m.build_opts("%s/idx%d" % (d, next(runs)), synth=(4, 5, 30000, 77, 0.03), conversion_table=conv, taxonomy_tree=nodes,
                                   name_table=names))
    assert_cycles_return_memory(cycle)


def test_hooks():
    m = capi()
    ix = m.Index(util.golden_index("adv"), 0)
    rng = np.random.default_rng(1)
    rows = rng.integers(0, int(ix.info.len) + 1, size=20000).astype(np.uint64)
    chars = rng.integers(0, 5, size=len(rows)).astype(np.uint8)

    def cycle():
        m.gather_rate(ix, 0, 1 << 22, 2, 2)
        m.test_lf(ix, rows, chars)
        m.test_resolve(ix, rows)
    assert_cycles_return_memory(cycle)
    ix.close()
