"""gzip input on the device: the inflater through the C ABI (cfb_gunzip_*) against zlib, and `centrifuge-class` on
.gz read files, which must write the bytes it writes for the same files uncompressed (and so the reference's)."""
import atexit
import gzip
import json
import os
import re
import struct
import subprocess
import zlib

import numpy as np
import pytest

import util
from test_gpu_text import decorate, write_fq

pytestmark = pytest.mark.gpu

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
CFB_EDATA = -7


def capi():
    from centrifuge_b200 import capi as c
    return c


def inflate(data, chunk_kb=0, piece=None, out_cap=1 << 24):
    g = capi().Gunzip(0, chunk_kb)
    try:
        return g.decompress(data, piece, out_cap), g.stats()
    finally:
        g.close()


def member(payload, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=(), header=None):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    parts, pos = [], 0
    for at, mode in flushes:
        parts += [c.compress(payload[pos:at]), c.flush(mode)]
        pos = at
    parts += [c.compress(payload[pos:]), c.flush()]
    hdr = header if header is not None else b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03"
    return hdr + b"".join(parts) + struct.pack("<II", zlib.crc32(payload), len(payload) & 0xffffffff)


def fastq(n, seed, lo=60, hi=160):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi))
        seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, L)].tobytes()
        out.append(b"@r%d\n%s\n+\n%s\n" % (i, seq, rng.integers(35, 74, L, dtype=np.uint8).tobytes()))
    return b"".join(out)


def mixed(seed):
    rng = np.random.default_rng(seed)
    return fastq(6000, seed) + rng.integers(0, 256, 80000, dtype=np.uint8).tobytes() + b"ACGT" * 60000 + bytes(150000) + fastq(3000, seed + 1)


CASES = ([("level%d" % lv, dict(level=lv)) for lv in (0, 1, 6, 9)]
         + [(n, dict(strategy=getattr(zlib, n))) for n in ("Z_FILTERED", "Z_HUFFMAN_ONLY", "Z_RLE", "Z_FIXED")]
         + [("sync_flush", dict(flushes=[(50000, zlib.Z_SYNC_FLUSH), (50001, zlib.Z_SYNC_FLUSH), (300000, zlib.Z_SYNC_FLUSH)])),
            ("full_flush", dict(flushes=[(70000, zlib.Z_FULL_FLUSH), (400000, zlib.Z_FULL_FLUSH)]))])


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_zlib_matrix_at_several_chunk_sizes_and_pieces(name, kw):
    data = mixed(len(name))
    gz = member(data, **kw)
    assert zlib.decompress(gz, 31) == data
    for chunk_kb, piece in ((1, None), (3, 7777), (64, None), (17, 100000)):
        got, st = inflate(gz, chunk_kb, piece, out_cap=1 << 20)
        assert got == data, (name, chunk_kb, piece)
        assert st["members"] == 1 and st["bytes_in"] == len(gz) and st["bytes_out"] == len(data)


def test_member_layouts_and_header_flags():
    a, b = fastq(2000, 1), fastq(500, 2)
    flags = 0x01 | 0x02 | 0x04 | 0x08 | 0x10
    h = b"\x1f\x8b\x08" + bytes([flags]) + b"\x00" * 6 + struct.pack("<H", 5) + b"AB\x01\x00z" + b"name.fq\x00" + b"a comment\x00"
    h += struct.pack("<H", zlib.crc32(h) & 0xffff)
    bgzf_eof = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
    def bgzf(payload):
        blocks = []
        for i in range(0, len(payload), 60000):
            body = member(payload[i:i + 60000])[10:]
            blocks.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", 18 + len(body) - 1) + body)
        return b"".join(blocks) + bgzf_eof
    files = {
        "multi": (member(a) + member(b) + member(a, level=1), a + b + a, 3),
        "empty_members": (member(b"") + member(a) + member(b"") + member(b""), a, 4),
        "only_empty": (member(b""), b"", 1),
        "all_flags": (member(a, header=h) + member(b, header=h), a + b, 2),
        "bgzf": (bgzf(a + b), a + b, None),
        "one_byte": (member(b"x"), b"x", 1),
    }
    for k, (gz, want, members) in files.items():
        assert gzip.decompress(gz) == want, k
        for chunk_kb in (1, 64):
            got, st = inflate(gz, chunk_kb, piece=5000)
            assert got == want, k
            if members is not None:
                assert st["members"] == members, (k, st)
    assert inflate(b"")[0] == b""


def test_sizes_around_chunk_multiples():
    rng = np.random.default_rng(5)
    for n in (0, 1, 1024 - 30, 2048 - 29, 2048 - 27, 3 * 1024 + 1, 64 * 1024 - 23, 64 * 1024 - 24):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        gz = member(data, level=0)
        got, _ = inflate(gz, 1)
        assert got == data, n
    for n in (1023, 1024, 1025, 2047, 2048, 2049):
        data = fastq(n, n)
        assert inflate(member(data), 1)[0] == data


def fixed_huffman(tokens):
    """raw DEFLATE, one final fixed-Huffman block: tokens are ints (literals) or (length, distance)"""
    bits = []
    def put(v, n, rev=False):
        if rev:
            v = int(format(v, "0%db" % n)[::-1], 2)
        bits.extend((v >> i) & 1 for i in range(n))
    def lit(s):
        if s < 144: put(0x30 + s, 8, True)
        elif s < 256: put(0x190 + s - 144, 9, True)
        elif s < 280: put(s - 256, 7, True)
        else: put(0xc0 + s - 280, 8, True)
    lb = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
    le = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    db = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577]
    de = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
    put(1, 1); put(1, 2)
    for t in tokens:
        if isinstance(t, int):
            lit(t)
            continue
        L, D = t
        s = max(i for i in range(29) if lb[i] <= L)
        lit(257 + s); put(L - lb[s], le[s])
        d = max(i for i in range(30) if db[i] <= D)
        put(d, 5, True); put(D - db[d], de[d])
    lit(256)
    bits += [0] * (-len(bits) % 8)
    return bytes(sum(bits[i + k] << k for k in range(8)) for i in range(0, len(bits), 8))


def test_distance_32768_and_long_matches_across_chunks():
    rng = np.random.default_rng(8)
    head = rng.integers(0, 256, 40000, dtype=np.uint8).tobytes()
    tokens, data = list(head), bytearray(head)
    for k in range(300):
        L, D = (258, 32768) if k % 3 else (258, 1 + k)
        tokens.append((L, D))
        for _ in range(L):
            data.append(data[-D])
        tokens += [7, 9]; data += b"\x07\x09"
    raw = fixed_huffman(tokens)
    data = bytes(data)
    assert zlib.decompress(raw, -15) == data
    gz = b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03" + raw + struct.pack("<II", zlib.crc32(data), len(data))
    for chunk_kb in (1, 2, 5):
        assert inflate(gz, chunk_kb)[0] == data


def test_gzip_inside_stored_blocks_is_redecoded_correctly():
    inner = b"".join(member(fastq(300, s)) for s in range(40))
    gz = member(inner, level=0) + member(inner, level=0)
    got, st = inflate(gz, 1)
    assert got == inner + inner
    assert st["redone"] > 0, st


def test_random_bytes():
    rng = np.random.default_rng(9)
    data = rng.integers(0, 256, 3_000_000, dtype=np.uint8).tobytes()
    assert inflate(member(data), 4)[0] == data
    with pytest.raises(capi().CfbError) as e:
        inflate(data)
    assert e.value.code == CFB_EDATA


def test_truncation_and_bit_flips_are_errors():
    data = fastq(3000, 11)
    gz = member(data) + member(data[:5000])
    rng = np.random.default_rng(12)
    for cut in sorted(set([1, 5, 9, 10, 11, 50, len(gz) - 1, len(gz) - 4, len(gz) - 8, len(gz) - 9]) | set(int(x) for x in rng.integers(1, len(gz), 20))):
        with pytest.raises(capi().CfbError) as e:
            inflate(gz[:cut], 1)
        assert e.value.code == CFB_EDATA, cut
    errors = 0
    for t in range(60):
        b = bytearray(gz)
        i = int(rng.integers(10, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
        try:
            got, _ = inflate(bytes(b), 2)
            assert got == data + data[:5000], (t, i)       # a flip that changes nothing decoded (e.g. padding) is fine
        except capi().CfbError as e:
            assert e.code == CFB_EDATA
            errors += 1
    assert errors > 50
    with pytest.raises(capi().CfbError):
        inflate(member(data) + b"trailing")


def test_state_restores_into_another_inflater():
    data = fastq(30000, 13)
    gz = member(data)
    c = capi()
    g = c.Gunzip(0, 1)                         # 512 KB of compressed input per pass: several passes
    pos, out, snap = 0, b"", None
    while len(out) < len(data) // 2:
        got, used = g.run(gz[pos:], True, out_cap=50000)
        pos += used
        out += got
        if len(got) < 50000:
            snap = (g.state(), len(out))
    g.close()
    assert snap is not None
    s, at = snap
    assert s.out_offset == at
    h = c.Gunzip(0, 64)
    h.set_state(s)
    rest = b"".join(h.decompress_iter(gz[s.in_offset:]))
    h.close()
    assert data[:at] + rest == data


def test_isize_wraps_past_4_gib():
    n = (1 << 32) + 12345
    c = zlib.compressobj(1, zlib.DEFLATED, 31)
    piece = bytes(1 << 26)
    parts, left = [], n
    while left:
        k = min(left, len(piece))
        parts.append(c.compress(piece[:k]))
        left -= k
    parts.append(c.flush())
    gz = b"".join(parts)
    assert struct.unpack("<I", gz[-4:])[0] == n & 0xffffffff
    g = capi().Gunzip(0, 0)
    crc, total = 0, 0
    for out in g.decompress_iter(gz, out_cap=1 << 27):
        assert not out.strip(b"\x00")
        crc = zlib.crc32(out, crc)
        total += len(out)
    assert g.stats()["members"] == 1
    g.close()
    assert total == n and crc == struct.unpack("<I", gz[-8:-4])[0]


# ------------------------------------------------------------------------------ centrifuge-class on .gz files
def run_cli(args, tmp, tag, block=None, env=None, ok=True):
    e = dict(os.environ, CFB_TEXT_STATS="1")
    if block:
        e["CFB_TEXT_BLOCK"] = str(block)
    e.update(env or {})
    tsv, rep, kr = (str(tmp / (tag + x)) for x in (".tsv", ".rep", ".kr"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep, "--kreport-file", kr], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=e)
    err = p.stderr.decode()
    if not ok:
        return p.returncode, err
    assert p.returncode == 0, err
    m = re.search(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units", err)
    g = re.search(r"gunzip: (\d+) members, (\d+) bytes in, (\d+) bytes out, (\d+) chunks, (\d+) re-decoded", err)
    st = dict(text=int(m.group(1)), fallbacks=int(m.group(3)), host=int(m.group(4)), gz=g and [int(x) for x in g.groups()])
    return tuple(open(x, "rb").read() for x in (tsv, rep, kr)), st


# Recorded reference outputs of these cases: util.reference's scheme (digests of what the unmodified reference wrote,
# re-recorded with CFB_RECORD_REFERENCE=1) in a file of their own.
DIGESTS = os.path.join(util.GOLDEN, "gunzip_digests.json")
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
    key = "gpu_gunzip/" + key
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


def gzfile(path, data, **kw):
    with open(path, "wb") as f:
        f.write(member(data, **kw))
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


def check_same(tmp, plain_args, gz_args, key, block, reads, extra_env=None):
    """the .gz run writes what the plain run writes, and the plain run what the reference writes"""
    want = run_ref(key, reference_args(plain_args), tmp)
    got_p, st_p = run_cli(plain_args, tmp, "plain", block)
    got_g, st_g = run_cli(gz_args, tmp, "gz", block, extra_env)
    util.assert_matches(got_p[:2], want, key)
    assert got_g == got_p, key
    assert st_g["gz"] and st_g["gz"][2] > 0
    return st_p, st_g


def test_cli_fastq_se_and_several_files(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(21)
    reads = decorate(util.synth.sample_reads(seqs, 2500, 60, seed=11, lens=(1, 120)) + util.synth.sample_reads(seqs, 2500, 150, seed=12, lens=(100, 300)), rng)
    fq = str(tmp_path / "r.fq")
    write_fq(fq, reads, rng, tail_newline=False)
    data = open(fq, "rb").read()
    fqz = gzfile(str(tmp_path / "r.fq.gz"), data)
    for chunk in ("1", "64"):
        st_p, st_g = check_same(tmp_path, ["-q", "-x", base, "-U", fq], ["-q", "-x", base, "-U", fqz], "fastq_se", 100000, len(reads), {"CFB_GZ_CHUNK_KB": chunk})
        assert st_g["fallbacks"] == 0 and st_g["host"] == 0 and st_g["text"] == len(reads), st_g
    # several files in one -U list, gzip and plain mixed
    args_p = ["-q", "-x", base, "-U", ",".join([fq, fq, fq])]
    args_g = ["-q", "-x", base, "-U", ",".join([fqz, fq, fqz])]
    check_same(tmp_path, args_p, args_g, "fastq_se_list", 100000, 3 * len(reads))
    # the record-level reader on gzip input: --host-parse, -s/-u
    for extra, key in ((["--host-parse"], "fastq_se"), (["-s", "100", "-u", "3000"], "fastq_se/-s 100 -u 3000")):
        st_p, st_g = check_same(tmp_path, ["-q", "-x", base, "-U", fq] + extra, ["-q", "-x", base, "-U", fqz] + extra, key, 100000, len(reads))
        assert st_g["text"] == 0


def test_cli_fastq_pe_gzip_and_mixed_mates(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(22)
    prs = util.synth.sample_pairs(seqs, 4000, 125, seed=31)
    f1, f2 = str(tmp_path / "p_1.fq"), str(tmp_path / "p_2.fq")
    write_fq(f1, decorate([(n, x) for n, x, _ in prs], rng), rng)
    write_fq(f2, [(n + "/2", y) for n, _, y in prs], rng)
    z1, z2 = gzfile(f1 + ".gz", open(f1, "rb").read()), gzfile(f2 + ".gz", open(f2, "rb").read(), level=1)
    for a, b in ((z1, z2), (z1, f2), (f1, z2)):
        _, st = check_same(tmp_path, ["-q", "-x", base, "-1", f1, "-2", f2], ["-q", "-x", base, "-1", a, "-2", b], "fastq_pe", 150000, len(prs))
        assert st["fallbacks"] == 0 and st["text"] == len(prs), st


def test_cli_fasta_across_span_cuts(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(23)
    reads = util.synth.sample_reads(seqs, 4000, 100, seed=5, lens=(20, 200))
    fa = str(tmp_path / "r.fa")
    data = b"".join(b">" + n.encode() + b"\n" + a.tobytes() + b"\n" for n, a in reads)
    open(fa, "wb").write(data)
    faz = gzfile(fa + ".gz", data, level=9)
    _, st = check_same(tmp_path, ["-f", "-x", base, "-U", fa], ["-f", "-x", base, "-U", faz], "fasta_se", 20000, len(reads), {"CFB_GZ_CHUNK_KB": "2"})
    assert st["fallbacks"] == 0 and st["text"] == len(reads), st


def test_cli_crlf_inside_gzip_falls_back(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 3000, 100, seed=21, lens=(40, 140))
    recs = [b"@" + n.encode() + b"\n" + a.tobytes() + b"\n+\n" + b"F" * len(a) + b"\n" for n, a in reads]
    recs[2000] = recs[2000].replace(b"\n", b"\r\n")
    fq = str(tmp_path / "c.fq")
    open(fq, "wb").write(b"".join(recs))
    fqz = gzfile(fq + ".gz", b"".join(recs))
    _, st = check_same(tmp_path, ["-q", "-x", base, "-U", fq], ["-q", "-x", base, "-U", fqz], "crlf", 60000, len(reads))
    assert st["fallbacks"] == 1 and st["text"] > 1000 and st["text"] + st["host"] == len(reads), st


def test_cli_corrupt_gzip_is_an_error(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 3000, 100, seed=2)
    data = b"".join(b"@" + n.encode() + b"\n" + a.tobytes() + b"\n+\n" + b"F" * len(a) + b"\n" for n, a in reads)
    good = member(data)
    bad_crc = good[:-8] + struct.pack("<I", zlib.crc32(data) ^ 1) + good[-4:]
    for tag, blob in (("truncated", good[: len(good) * 2 // 3]), ("crc", bad_crc), ("trailing", good + b"junk")):
        path = str(tmp_path / (tag + ".fq.gz"))
        open(path, "wb").write(blob)
        for extra in ([], ["--host-parse"]):
            rc, err = run_cli(["-q", "-x", base, "-U", path] + extra, tmp_path, tag, 60000, ok=False)
            assert rc == 1 and ("Error: %s: " % path) in err, (tag, err)
    # a file that starts with 1f but is not gzip keeps today's reader error
    path = str(tmp_path / "x.fq")
    open(path, "wb").write(b"\x1f\x00" + data)
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
    fqz = gzfile(fq + ".gz", open(fq, "rb").read())
    check_same(tmp_path, ["-q", "-x", base, "-U", fq, "--devices", "0,1"], ["-q", "-x", base, "-U", fqz, "--devices", "0,1"], "devices", 50000, len(reads))
