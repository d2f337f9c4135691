"""GPU: units with a mate longer than 60 000 bases (long units) are searched in parallel segments and classified with the
records the oracle gives, in unit order among short units, through the byte, packed and resident forms."""
import atexit
import bz2
import ctypes as C
import gzip
import json
import os
import re
import subprocess

import numpy as np
import pytest

import util
from test_gpu_parity import assert_same, to_cbatch

pytestmark = pytest.mark.gpu

OPTIONS = {"k5": {}, "k1": dict(k=1), "minhit15": dict(min_hitlen=15), "host": dict(k=2, host=(100, 1005)),
           "excl": dict(excl=(1003,)), "genus": dict(rank_slot=2), "notraverse": dict(traverse=False)}


def syn_big():
    return util.build_index("syn_big", 10, 10, 300000, seed=3), util.synth.make_genomes(10, 10, 300000, 3)


def chimera(seqs, length, rng, sub=0.01):
    """Pieces of several genomes from both strands (codes 0..3), ~sub substitutions and a few Ns."""
    out, have = [], 0
    while have < length:
        s = seqs[int(rng.integers(len(seqs)))]
        n = min(int(rng.integers(2000, 120000)), len(s), length - have)
        p = int(rng.integers(0, len(s) - n + 1))
        piece = s[p:p + n].copy()
        if rng.random() < 0.5:
            piece = (3 - piece)[::-1]
        out.append(piece); have += n
    r = np.concatenate(out)
    m = rng.random(length) < sub
    r[m] = (r[m] + 1) & 3
    a = util.synth.ACGT[r].copy()
    a[rng.random(length) < 0.0005] = ord("N")
    return a


def exact(seqs, si, p, n, rc=False):
    r = seqs[si][p:p + n]
    return util.synth.ACGT[(3 - r)[::-1] if rc else r].copy()


def short_reads(seqs, n, seed):
    return [a for _, a in util.synth.sample_reads(seqs, n, 150, seed=seed, lens=(60, 400))]


def single_reads(seqs):
    rng = np.random.default_rng(1)
    longs = [exact(seqs, 3, 1000, 60001), exact(seqs, 17, 5000, 65551, rc=True), exact(seqs, 42, 100, 70000),
             chimera(seqs, 300000, rng), chimera(seqs, 1000000, rng, sub=0.02)]
    reads = short_reads(seqs, 120, 5)
    for i, a in enumerate(longs):
        reads.insert(10 + 20 * i, a)
    return reads


def single_batch(seqs):
    return util.Batch(single_reads(seqs))


def paired_batch(seqs):
    rng = np.random.default_rng(2)
    m1 = short_reads(seqs, 40, 6); m2 = short_reads(seqs, 40, 7)
    for i in (3, 11, 30):                      # only mate 2 long
        m2[i] = chimera(seqs, 61000 + 1000 * i, rng)
    m1[20] = exact(seqs, 55, 2000, 66000); m2[20] = exact(seqs, 55, 80000, 62000, rc=True)
    return util.Batch(m1, m2)


@pytest.fixture(scope="module")
def fixture():
    base, seqs = syn_big()
    o = util.Oracle(base)
    yield base, seqs, o
    o.close()


@pytest.mark.parametrize("opt", sorted(OPTIONS))
def test_long_units_match_oracle(fixture, opt):
    from centrifuge_b200 import capi as m
    base, seqs, o = fixture
    ix = m.Index(base, 0); ctx = m.Context(ix, m.make_params(**OPTIONS[opt]))
    for b in (single_batch(seqs), paired_batch(seqs)):
        on, orec, _ = o.classify(b, util.make_oparams(**OPTIONS[opt]))
        off, recs = ctx.classify(to_cbatch(b))
        assert_same(on, orec, np.diff(off.astype(np.int64)).astype(np.uint32), recs)
    st = ctx.long_stats()
    assert st["units"] == 9 and st["segment_searches"] > 0          # 5 + 4 long units went through the segmented path
    ctx.close(); ix.close()


def test_wrapped_score_is_never_observed(fixture):
    """An exact 70 kb read: its single hit's score (len - 15)^2 wraps in 32 bits, as in the reference."""
    from centrifuge_b200 import capi as m
    base, seqs, o = fixture
    b = util.Batch([exact(seqs, 42, 100, 70000)])
    on, orec, _ = o.classify(b, util.make_oparams())
    ix = m.Index(base, 0); ctx = m.Context(ix)
    off, recs = ctx.classify(to_cbatch(b))
    assert_same(on, orec, np.diff(off.astype(np.int64)).astype(np.uint32), recs)
    assert len(recs) and int(recs["hitlen"].max()) >= 70000
    ctx.close(); ix.close()


def test_packed_and_resident_forms(fixture):
    from centrifuge_b200 import capi as m
    base, seqs, _ = fixture
    ix = m.Index(base, 0); ctx = m.Context(ix)
    for b in (single_batch(seqs), paired_batch(seqs)):
        cb = to_cbatch(b)
        off0, rec0 = ctx.classify(cb)
        words, npos = m.pack_batch(cb)
        len2, flags = (b.len2, b.flags & 3) if b.paired else (None, b.flags & 1)
        ctx.submit_packed(1, m.make_batch_packed(words, b.len1, len2, npos, flags.astype(np.uint8)))
        off1, rec1 = ctx.wait(1)
        assert np.array_equal(off0, off1) and np.array_equal(rec0, rec1)
        d = ctx.upload(cb)
        ctx.classify_resident(d)
        off2, rec2 = ctx.resident_result()
        assert np.array_equal(off0, off2) and np.array_equal(rec0, rec2)
        half = b.n // 2                          # a window that holds part of the long units
        ctx.classify_resident(d, half, b.n - half)
        off3, rec3 = ctx.resident_result()
        assert np.array_equal(rec3, rec0[off0[half]:]) and np.array_equal(off3.astype(np.int64), off0[half:].astype(np.int64) - int(off0[half]))
        m.lib().cfb_dbatch_free(ctx.h, d)
    ctx.close(); ix.close()


def test_short_units_are_unchanged_by_long_ones(fixture):
    from centrifuge_b200 import capi as m
    base, seqs, _ = fixture
    reads = single_reads(seqs)
    b = util.Batch(reads)
    keep = [i for i in range(b.n) if len(reads[i]) <= 60000]
    ix = m.Index(base, 0); ctx = m.Context(ix)
    off, recs = ctx.classify(to_cbatch(b))
    sub = util.Batch([reads[i] for i in keep])
    off_s, recs_s = ctx.classify(to_cbatch(sub))
    got = np.concatenate([recs[off[i]:off[i + 1]] for i in keep])
    assert np.array_equal(got, recs_s)
    assert np.array_equal(np.diff(off.astype(np.int64))[keep], np.diff(off_s.astype(np.int64)))
    ctx.close(); ix.close()


def test_mate_over_the_limit_is_rejected(fixture):
    """A batch header claiming a 2^31-base mate: CFB_EINVAL with the limit in the message, before any base is read."""
    from centrifuge_b200 import capi as m
    base, _, _ = fixture
    ix = m.Index(base, 0); ctx = m.Context(ix)
    bases = np.zeros(16, dtype=np.uint8)
    off = np.zeros(1, dtype=np.uint64); ln = np.array([2 ** 31], dtype=np.uint32)
    res = (C.c_uint64 * 4)()
    rc = m.lib().cfb_classify_batch(ctx.h, C.byref(m.make_batch(bases, off, ln)), res)
    assert rc == -1 and b"2147483647" in m.lib().cfb_last_error()
    ctx.close(); ix.close()


# ------------------------------------------------------------------------------ centrifuge-class on files with long reads
EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
DIGESTS = os.path.join(util.GOLDEN, "long_read_digests.json")
_recorded = {}


def _save_digests():
    old = {}
    if os.path.exists(DIGESTS):
        with open(DIGESTS) as f:
            old = json.load(f)
    old.update(_recorded)
    with open(DIGESTS, "w") as f:
        json.dump(old, f, indent=0, sort_keys=True)
        f.write("\n")


def ref_digest(key, args, tmp):
    """digest of the reference's (TSV, report) for these arguments, recorded with CFB_RECORD_REFERENCE=1"""
    key = "gpu_ultra_long/" + key
    if util.RECORD:
        if not util.have_ref():
            raise RuntimeError("CFB_RECORD_REFERENCE=1 needs the reference binaries under oracle/_ref (make -C oracle ref)")
        if not _recorded:
            atexit.register(_save_digests)
        _recorded[key] = util.digest(util.run_cli(util.REF_CLASS, args, str(tmp / "ref.tsv"), str(tmp / "ref.rep")))
        return _recorded[key]
    with open(DIGESTS) as f:
        digests = json.load(f)
    if key not in digests:
        raise KeyError("no recorded reference output for %r (re-record with CFB_RECORD_REFERENCE=1)" % key)
    return digests[key]


def run_cli(args, tmp, tag):
    tsv, rep, kr = (str(tmp / (tag + x)) for x in (".tsv", ".rep", ".kr"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep, "--kreport-file", kr], stdout=subprocess.DEVNULL,
                       stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
    err = p.stderr.decode()
    assert p.returncode == 0, err
    m = re.search(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units", err)
    lu = re.search(r"long units: (\d+) \((\d+) bases\), (\d+) partial searches in segment chains, (\d+) re-searched", err)
    st = dict(text=int(m.group(1)), fallbacks=int(m.group(3)), host=int(m.group(4)), long=int(lu.group(1)))
    return tuple(open(x, "rb").read() for x in (tsv, rep, kr)), st


def cli_reads(seqs):
    """short reads with long ones among them: a 60 001 base read, exact reads whose single hit's score wraps, and chimeras"""
    rng = np.random.default_rng(8)
    reads = [("s%d" % i, a) for i, a in enumerate(short_reads(seqs, 150, 9))]
    longs = [("l60001", exact(seqs, 3, 1000, 60001)), ("l65551_wrap", exact(seqs, 17, 5000, 65551, rc=True)),
             ("l90000_wrap", exact(seqs, 64, 20000, 90000)), ("l300k", chimera(seqs, 300000, rng))]
    for i, r in enumerate(longs):
        reads.insert(7 + 30 * i, r)
    return reads


@pytest.fixture(scope="module")
def cli_files(fixture, tmp_path_factory):
    base, seqs, _ = fixture
    d = tmp_path_factory.mktemp("longcli")
    reads = cli_reads(seqs)
    fq, fa = str(d / "r.fq"), str(d / "r.fa")
    util.synth.write_fastq(fq, reads)
    util.synth.write_fasta(fa, reads)
    for p in (fq, fa):
        data = open(p, "rb").read()
        with open(p + ".gz", "wb") as f:
            f.write(gzip.compress(data, 6))
        with open(p + ".bz2", "wb") as f:
            f.write(bz2.compress(data, 9))
    return base, fq, fa


@pytest.mark.parametrize("fmt", ["fq", "fa"])
def test_cli_long_reads_match_reference(cli_files, tmp_path, fmt):
    base, fq, fa = cli_files
    path, flag = (fq, "-q") if fmt == "fq" else (fa, "-f")
    want = ref_digest(fmt, [flag, "-x", base, "-U", path], tmp_path)
    got, st = run_cli([flag, "-x", base, "-U", path], tmp_path, "plain")
    util.assert_matches(got[:2], want, fmt)
    assert st["fallbacks"] == 0 and st["host"] == 0 and st["text"] == 154 and st["long"] == 4, st
    for ext in (".gz", ".bz2"):
        got_c, st_c = run_cli([flag, "-x", base, "-U", path + ext], tmp_path, ext[1:])
        assert got_c == got and st_c["fallbacks"] == 0, ext
    got_h, st_h = run_cli([flag, "-x", base, "-U", path, "--host-parse"], tmp_path, "host")
    assert got_h == got and st_h["host"] == 154


def test_cli_long_reads_sequence_columns(cli_files, tmp_path):
    """readSeq / readQual rows of long reads come out of the device formatter as the record-level path writes them"""
    base, fq, _ = cli_files
    cols = ["--tab-fmt-cols", "readID,seqID,taxID,score,hitLength,queryLength,numMatches,readSeq,readQual"]
    got, st = run_cli(["-q", "-x", base, "-U", fq] + cols, tmp_path, "cols")
    got_h, _ = run_cli(["-q", "-x", base, "-U", fq, "--host-parse"] + cols, tmp_path, "cols_host")
    assert st["fallbacks"] == 0 and st["host"] == 0
    assert got == got_h
    assert max(len(x) for x in got[0].split(b"\n")) > 2 * 300000
