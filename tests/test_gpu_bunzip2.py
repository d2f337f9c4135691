"""bzip2 input on the device: the decompressor through the C ABI (cfb_bunzip2_*) against Python's bz2, and
`centrifuge-class` on .bz2 read files, which must write the bytes it writes for the same files uncompressed (and so the
reference's)."""
import atexit
import bz2
import gzip
import json
import os
import re
import subprocess

import numpy as np
import pytest

import util
import util_bzip2 as ub
from test_bunzip2_host import fasta, fastq, magic_block
from test_gpu_text import decorate, write_fq

pytestmark = pytest.mark.gpu

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
CFB_EDATA = -7


def capi():
    from centrifuge_b200 import capi as c
    return c


def bunzip2(data, pass_kb=0, piece=None, out_cap=1 << 24):
    g = capi().Bunzip2(0, pass_kb)
    try:
        return g.decompress(data, piece, out_cap), g.stats()
    finally:
        g.close()


def pbzip2(data, level=9, piece=900000):
    """one stream per piece, as pbzip2 writes"""
    return b"".join(bz2.compress(data[i:i + piece], level) for i in range(0, len(data), piece)) or bz2.compress(b"", level)


def payloads():
    rng = np.random.default_rng(1)
    runs = b"".join(bytes([65 + i % 20]) * k + b"x" for i, k in enumerate((3, 4, 5, 259, 260, 1000, 4, 3, 8, 255, 256, 257, 258)))
    return {
        "fastq": fastq(12000, 1),
        "fasta": fasta(3000, 2),
        "random": rng.integers(0, 256, 1_200_000, dtype=np.uint8).tobytes(),
        "all_bytes": bytes(range(256)) * 7,
        "one_byte": b"Q",
        "runs": runs * 20,
        "periodic_ab": b"ab" * 50000,
        "periodic_record": b"@r\nACGTACGTTT\n+\nFFFFFFFFFF\n" * 40000,
        "mixed": fastq(3000, 3) + bytes(2_000_000) + rng.integers(0, 256, 300000, dtype=np.uint8).tobytes() + b"ACGT" * 200000,
    }


@pytest.mark.parametrize("name", list(payloads()))
def test_matches_bz2_at_several_pass_sizes_pieces_and_out_caps(name):
    data = payloads()[name]
    for level in (1, 9):
        comp = bz2.compress(data, level)
        for pass_kb, piece, out_cap in ((1, None, 1 << 24), (7, 7777, 100000), (256, 100000, 1 << 20), (0, None, 1 << 24)):
            got, st = bunzip2(comp, pass_kb, piece, out_cap)
            assert got == data, (name, level, pass_kb, piece)
            assert st["streams"] == 1 and st["bytes_in"] == len(comp) and st["bytes_out"] == len(data) and st["trailing"] == 0, st


def test_every_level_concatenated_empty_and_pbzip2_streams():
    data = fastq(30000, 4)
    for level in range(1, 10):
        comp = bz2.compress(data, level)
        got, st = bunzip2(comp, 64)
        assert got == data, level
        assert st["blocks"] >= len(data) // (level * 100000 + 1)
    empty = bz2.compress(b"")
    assert bunzip2(empty)[0] == b""
    assert bunzip2(b"")[0] == b""
    parts = [bz2.compress(data[:5000], 1), empty, bz2.compress(data, 9), empty, empty, bz2.compress(b"x", 3)]
    got, st = bunzip2(b"".join(parts), 2, 3000)
    assert got == data[:5000] + data + b"x" and st["streams"] == 6
    comp = pbzip2(data)
    for pass_kb in (1, 300, 0):
        got, st = bunzip2(comp, pass_kb, out_cap=1 << 20)
        assert got == data and st["streams"] == -(-len(data) // 900000)


def test_full_random_block_and_pass_smaller_than_a_block():
    rng = np.random.default_rng(5)
    data = rng.integers(0, 256, 899000, dtype=np.uint8).tobytes() + fastq(8000, 5)
    comp = bz2.compress(data, 9)
    for pass_kb, piece in ((1, None), (1, 50000), (100, 333333)):
        assert bunzip2(comp, pass_kb, piece)[0] == data


def test_one_gib_of_zeros_through_a_16_mb_out_cap():
    c = bz2.BZ2Compressor(9)
    piece = bytes(1 << 26)
    comp = b"".join(c.compress(piece) for _ in range(16)) + c.flush()
    assert len(comp) < 4096
    g = capi().Bunzip2(0, 0)
    total, calls = 0, 0
    for out in g.decompress_iter(comp, out_cap=16 << 20):
        assert len(out) <= 16 << 20 and not out.strip(b"\x00")
        total += len(out)
        calls += 1
    st = g.stats()
    g.close()
    assert total == 1 << 30 and calls >= 64 and st["blocks"] >= 23, (total, st)


def test_block_magic_inside_coded_data_is_a_rejected_start():
    blk, out = magic_block()
    more = fastq(2000, 6)
    comp = ub.stream([blk]) + bz2.compress(more)
    assert bz2.decompress(comp) == out + more
    for pass_kb in (1, 0):
        got, st = bunzip2(comp, pass_kb)
        assert got == out + more and st["rejected"] >= 1, st


def expect_edata(comp, pass_kb=0, what=None):
    with pytest.raises(capi().CfbError) as e:
        bunzip2(comp, pass_kb)
    assert e.value.code == CFB_EDATA, str(e.value)
    if what:
        assert what in str(e.value), str(e.value)


def crafted(**kw):
    data = fastq(40, 8)
    L, orig = ub.bwt(ub.rle1(data))
    syms, used = ub.mtf_symbols(L)
    blk = dict(syms=syms, used=used, orig_ptr=orig, out=data, n_groups=2)
    blk.update(kw)
    return ub.stream([blk])


def test_corrupt_streams_are_errors():
    data = fastq(3000, 11)
    comp = bz2.compress(data, 1) + bz2.compress(data[:5000], 3)
    rng = np.random.default_rng(12)
    for cut in sorted(set([1, 3, 4, 9, 10, 11, 50, len(comp) - 1, len(comp) - 4, len(comp) - 10]) | set(int(x) for x in rng.integers(1, len(comp), 12))):
        expect_edata(comp[:cut], 1)
    errors = 0
    for t in range(40):
        b = bytearray(comp)
        i = int(rng.integers(4, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
        try:
            got, _ = bunzip2(bytes(b), 2)
            assert got == data + data[:5000], (t, i)
        except capi().CfbError as e:
            assert e.code == CFB_EDATA
            errors += 1
    assert errors > 35
    expect_edata(crafted(randomised=1), what="randomised")
    expect_edata(crafted(crc=123), what="block CRC")
    good = crafted()
    expect_edata(good[:-4] + bytes([good[-4] ^ 1]) + good[-3:], what="stream CRC")
    expect_edata(crafted(orig_ptr=(1 << 24) - 1), what="origPtr")
    expect_edata(crafted(start_len=21), what="code lengths")
    expect_edata(crafted(selectors=[0, 2]), what="selectors")
    expect_edata(crafted(n_selectors=0), what="selectors")
    expect_edata(b"BZh1" + bz2.compress(rng.integers(0, 256, 150000, dtype=np.uint8).tobytes(), 9)[4:], what="longer than its level")
    expect_edata(b"BZh9" + b"x" * 100)


def test_padded_code_lengths_are_an_error_in_any_piece_size():
    """8 MB of +1/-1 code-length steps after a valid block header: an error, never a decoder waiting for more input"""
    comp = ub.padded_lengths_stream(8 << 20)
    for piece, out_cap in ((None, 1 << 24), (1 << 20, 1 << 16), (64 << 20, 1 << 24)):
        with pytest.raises(capi().CfbError) as e:
            bunzip2(comp, 0, piece, out_cap)
        assert e.value.code == CFB_EDATA and "code lengths" in str(e.value), str(e.value)
    g = capi().Bunzip2(0, 0)                   # fed as the CLI's reader feeds it: a first call that is not the last
    with pytest.raises(capi().CfbError):
        g.run(comp[: 4 << 20], False)
    g.close()


def test_trailing_garbage_is_ignored_and_counted():
    data = fastq(3000, 13)
    comp = bz2.compress(data)
    for tail in (b"garbage", b"\0" * 1000, b"BZhx", b"BZh0", b"x" * 5000):
        for pass_kb in (1, 0):
            got, st = bunzip2(comp + tail, pass_kb, piece=4000)
            assert got == data and st["trailing"] == len(tail) and st["streams"] == 1, (tail, st)
    # a following header starts a stream whose errors are errors; so does the end of the file inside "BZh[1-9]"
    # (`bzip2 -dc` 1.0.8: "file ends unexpectedly")
    for tail in (b"BZh9" + b"x" * 20, b"BZh9", b"B", b"BZ", b"BZh"):
        expect_edata(comp + tail)


# ------------------------------------------------------------------------------ centrifuge-class on .bz2 files
def run_cli(args, tmp, tag, block=None, env=None, ok=True):
    e = dict(os.environ, CFB_TEXT_STATS="1")
    if block:
        e["CFB_TEXT_BLOCK"] = str(block)
    e.update(env or {})
    tsv, rep, kr = (str(tmp / (tag + x)) for x in (".tsv", ".rep", ".kr"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep, "--kreport-file", kr], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=e,
                       timeout=600)
    err = p.stderr.decode()
    if not ok:
        return p.returncode, err
    assert p.returncode == 0, err
    m = re.search(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units", err)
    b = re.search(r"bunzip2: (\d+) streams, (\d+) bytes in, (\d+) bytes out, (\d+) blocks, (\d+) rejected block starts", err)
    st = dict(text=int(m.group(1)), fallbacks=int(m.group(3)), host=int(m.group(4)), bz=b and [int(x) for x in b.groups()], err=err)
    return tuple(open(x, "rb").read() for x in (tsv, rep, kr)), st


# Recorded reference outputs of these cases: util.reference's scheme (digests of what the unmodified reference wrote,
# re-recorded with CFB_RECORD_REFERENCE=1) in a file of their own.
DIGESTS = os.path.join(util.GOLDEN, "bunzip2_digests.json")
_recorded = {}


def _save_digests():
    with open(DIGESTS) as f:
        old = json.load(f)
    old.update(_recorded)
    with open(DIGESTS, "w") as f:
        json.dump(old, f, indent=0, sort_keys=True)
        f.write("\n")


def run_ref(key, args, tmp):
    """digest of the reference's (TSV, report) for these arguments"""
    key = "gpu_bunzip2/" + key
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


def bzfile(path, data, level=9):
    with open(path, "wb") as f:
        f.write(bz2.compress(data, level))
    return path


def gzfile(path, data):
    with open(path, "wb") as f:
        f.write(gzip.compress(data, 6))
    return path


@pytest.fixture(scope="module")
def syn():
    base = util.build_index("syn_a", 5, 4, 60000, seed=7, strains=True)
    return base, util.synth.make_genomes(5, 4, 60000, 7)


def reference_args(args):
    """the reference's command for ours: options of this project only (--host-parse, --devices) left out"""
    out, skip = [], False
    for a in args:
        if skip:
            skip = False
        elif a == "--devices":
            skip = True
        elif a != "--host-parse":
            out.append(a)
    return out


def check_same(tmp, plain_args, bz_args, key, block, extra_env=None):
    """the .bz2 run writes what the plain run writes, and the plain run what the reference writes"""
    want = run_ref(key, reference_args(plain_args), tmp)
    got_p, st_p = run_cli(plain_args, tmp, "plain", block)
    got_b, st_b = run_cli(bz_args, tmp, "bz", block, extra_env)
    util.assert_matches(got_p[:2], want, key)
    assert got_b == got_p, key
    assert st_b["bz"] and st_b["bz"][2] > 0
    return st_p, st_b


def test_cli_fastq_se_and_several_files(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(21)
    reads = decorate(util.synth.sample_reads(seqs, 2500, 60, seed=11, lens=(1, 120)) + util.synth.sample_reads(seqs, 2500, 150, seed=12, lens=(100, 300)), rng)
    fq = str(tmp_path / "r.fq")
    write_fq(fq, reads, rng, tail_newline=False)
    data = open(fq, "rb").read()
    fqb = bzfile(str(tmp_path / "r.fq.bz2"), data, 1)
    fqz = gzfile(str(tmp_path / "r.fq.gz"), data)
    for pass_kb in ("1", "64"):
        st_p, st_b = check_same(tmp_path, ["-q", "-x", base, "-U", fq], ["-q", "-x", base, "-U", fqb], "fastq_se", 100000, {"CFB_BZ2_PASS_KB": pass_kb})
        assert st_b["fallbacks"] == 0 and st_b["host"] == 0 and st_b["text"] == len(reads), st_b
    # several files in one -U list: bzip2, gzip and plain mixed
    args_p = ["-q", "-x", base, "-U", ",".join([fq, fq, fq])]
    args_b = ["-q", "-x", base, "-U", ",".join([fqb, fqz, fq])]
    check_same(tmp_path, args_p, args_b, "fastq_se_list", 100000)
    # the record-level reader on bzip2 input: --host-parse, -s/-u
    for extra, key in ((["--host-parse"], "fastq_se"), (["-s", "100", "-u", "3000"], "fastq_se/-s 100 -u 3000")):
        st_p, st_b = check_same(tmp_path, ["-q", "-x", base, "-U", fq] + extra, ["-q", "-x", base, "-U", fqb] + extra, key, 100000)
        assert st_b["text"] == 0


def test_cli_fastq_pe_bzip2_and_mixed_mates(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(22)
    prs = util.synth.sample_pairs(seqs, 4000, 125, seed=31)
    f1, f2 = str(tmp_path / "p_1.fq"), str(tmp_path / "p_2.fq")
    write_fq(f1, decorate([(n, x) for n, x, _ in prs], rng), rng)
    write_fq(f2, [(n + "/2", y) for n, _, y in prs], rng)
    b1, b2 = bzfile(f1 + ".bz2", open(f1, "rb").read()), bzfile(f2 + ".bz2", open(f2, "rb").read(), 1)
    z2 = gzfile(f2 + ".gz", open(f2, "rb").read())
    for a, b in ((b1, b2), (b1, z2), (b1, f2), (f1, b2)):
        _, st = check_same(tmp_path, ["-q", "-x", base, "-1", f1, "-2", f2], ["-q", "-x", base, "-1", a, "-2", b], "fastq_pe", 150000)
        assert st["fallbacks"] == 0 and st["text"] == len(prs), st


def test_cli_fasta_across_span_cuts(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 4000, 100, seed=5, lens=(20, 200))
    fa = str(tmp_path / "r.fa")
    data = b"".join(b">" + n.encode() + b"\n" + a.tobytes() + b"\n" for n, a in reads)
    open(fa, "wb").write(data)
    fab = str(tmp_path / "r.fa.bz2")
    open(fab, "wb").write(pbzip2(data, 1, 100000))
    _, st = check_same(tmp_path, ["-f", "-x", base, "-U", fa], ["-f", "-x", base, "-U", fab], "fasta_se", 20000, {"CFB_BZ2_PASS_KB": "2"})
    assert st["fallbacks"] == 0 and st["text"] == len(reads), st


def test_cli_crlf_inside_bzip2_falls_back(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 3000, 100, seed=21, lens=(40, 140))
    recs = [b"@" + n.encode() + b"\n" + a.tobytes() + b"\n+\n" + b"F" * len(a) + b"\n" for n, a in reads]
    recs[2000] = recs[2000].replace(b"\n", b"\r\n")
    fq = str(tmp_path / "c.fq")
    open(fq, "wb").write(b"".join(recs))
    fqb = bzfile(fq + ".bz2", b"".join(recs))
    _, st = check_same(tmp_path, ["-q", "-x", base, "-U", fq], ["-q", "-x", base, "-U", fqb], "crlf", 60000)
    assert st["fallbacks"] == 1 and st["text"] > 1000 and st["text"] + st["host"] == len(reads), st


def test_cli_corrupt_bzip2_is_an_error_and_trailing_garbage_a_warning(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 3000, 100, seed=2)
    data = b"".join(b"@" + n.encode() + b"\n" + a.tobytes() + b"\n+\n" + b"F" * len(a) + b"\n" for n, a in reads)
    good = bz2.compress(data)
    bad_crc = good[:-6] + bytes([good[-6] ^ 0x10]) + good[-5:]
    for tag, blob in (("truncated", good[: len(good) * 2 // 3]), ("crc", bad_crc), ("header", good + b"BZh9junk")):
        path = str(tmp_path / (tag + ".fq.bz2"))
        open(path, "wb").write(blob)
        for extra in ([], ["--host-parse"]):
            rc, err = run_cli(["-q", "-x", base, "-U", path] + extra, tmp_path, tag, 60000, ok=False)
            assert rc == 1 and ("Error: %s: " % path) in err, (tag, err)
    fq = str(tmp_path / "t.fq")
    open(fq, "wb").write(data)
    path = str(tmp_path / "t.fq.bz2")
    open(path, "wb").write(good + b"trailing garbage\n")
    for extra in ([], ["--host-parse"]):
        got_p, _ = run_cli(["-q", "-x", base, "-U", fq] + extra, tmp_path, "tp", 60000)
        got_b, st = run_cli(["-q", "-x", base, "-U", path] + extra, tmp_path, "tb", 60000)
        assert got_b == got_p
        assert st["err"].count("Warning: %s: trailing garbage after the last bzip2 stream ignored" % path) == 1, st["err"]
    # the same file twice in one -U list: one warning for each
    got_p, _ = run_cli(["-q", "-x", base, "-U", ",".join([fq, fq])], tmp_path, "tp2", 60000)
    got_b, st = run_cli(["-q", "-x", base, "-U", ",".join([path, path])], tmp_path, "tb2", 60000)
    assert got_b == got_p and st["err"].count("Warning: %s: trailing garbage" % path) == 2, st["err"]
    # a valid header followed by 8 MB of padded code lengths: an error, not a reader that never returns
    path = str(tmp_path / "padded.fq.bz2")
    open(path, "wb").write(ub.padded_lengths_stream(8 << 20))
    for extra in ([], ["--host-parse"]):
        rc, err = run_cli(["-q", "-x", base, "-U", path] + extra, tmp_path, "pad", 60000, ok=False)
        assert rc == 1 and ("Error: %s: invalid code lengths" % path) in err, err
    # a file that starts with BZh9 but is not bzip2 keeps today's reader error
    path = str(tmp_path / "x.fq")
    open(path, "wb").write(b"BZh9" + data)
    rc, err = run_cli(["-q", "-x", base, "-U", path], tmp_path, "x", ok=False)
    assert rc == 1 and "does not look like a FASTQ file" in err


def test_cli_two_devices(syn, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    base, seqs = syn
    rng = np.random.default_rng(24)
    reads = decorate(util.synth.sample_reads(seqs, 3000, 100, seed=14, lens=(50, 150)), rng)
    fq = str(tmp_path / "d.fq")
    write_fq(fq, reads, rng)
    fqb = bzfile(fq + ".bz2", open(fq, "rb").read())
    check_same(tmp_path, ["-q", "-x", base, "-U", fq, "--devices", "0,1"], ["-q", "-x", base, "-U", fqb, "--devices", "0,1"], "devices", 50000)
