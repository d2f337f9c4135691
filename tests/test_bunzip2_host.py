"""The device bzip2 decompressor's per-block stages (centrifuge_b200/csrc/cf_bzip2.h), compiled for the host by
tests/native/bunzip2_host.cpp and checked against Python's bz2: every level, single, concatenated and empty streams,
FASTQ / FASTA / random / periodic data, runs around the RLE1 thresholds, every nGroups, a full 900 K block, truncations
and bit flips, and crafted blocks (tests/util_bzip2.py) for each malformed field and for a block magic inside a
block's coded data."""
import bz2
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import util
import util_bzip2 as ub

E_INPUT, E_MAGIC, E_RANDOMISED, E_MAP, E_GROUPS, E_SELECTORS, E_LENGTHS, E_CODE, E_SIZE, E_ORIGPTR, E_RLE = range(-1, -12, -1)
BLOCK_MAX = 900000


@pytest.fixture(scope="module")
def bz(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("bunzip2_host") / "bunzip2_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(util.ROOT, "tests", "native", "bunzip2_host.cpp")])
    lib = C.CDLL(so)
    lib.bzh_scan.restype = C.c_uint64
    lib.bzh_block_output.restype = C.c_int64
    lib.bzh_crc.restype = C.c_uint32
    return lib


def _buf(data):
    return np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)


def decode_block(lib, data, bit):
    buf = _buf(data)
    L = np.zeros(BLOCK_MAX, dtype=np.uint8)
    res = np.zeros(7, dtype=np.int64)
    lib.bzh_decode_block(buf.ctypes.data_as(C.c_void_p), C.c_uint64(len(data)), C.c_uint64(bit), L.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p))
    r = dict(zip(("status", "n", "orig_ptr", "crc", "end_bit", "n_groups", "n_selectors"), (int(x) for x in res)))
    return r, L[: max(0, r["n"])]


def block_output(lib, L, orig, seg=0):
    cap = max(64, len(L) * 260)
    out = np.zeros(cap, dtype=np.uint8)
    crc = C.c_uint32()
    k = lib.bzh_block_output(np.ascontiguousarray(L).ctypes.data_as(C.c_void_p), C.c_uint32(len(L)), C.c_uint32(orig), C.c_uint32(seg),
                             out.ctypes.data_as(C.c_void_p), C.c_uint64(cap), C.byref(crc))
    assert k != -3, "segmented RLE1 disagrees with its own chained start states"
    return (None if k < 0 else out[:k].tobytes()), crc.value


def scan(lib, data, lo=0, hi=None):
    hi = len(data) * 8 if hi is None else hi
    out = np.zeros(4096, dtype=np.int64)
    k = lib.bzh_scan(_buf(data).ctypes.data_as(C.c_void_p), C.c_uint64(len(data)), C.c_uint64(lo), C.c_uint64(hi), out.ctypes.data_as(C.c_void_p), C.c_uint64(len(out)))
    return [int(x) for x in out[:min(k, len(out))]]


class BzError(Exception):
    pass


def bits_at(data, b, k):
    v = int.from_bytes(data[b // 8: b // 8 + 16].ljust(16, b"\0"), "big")
    return (v >> (128 - (b % 8) - k)) & ((1 << k) - 1)


def decompress(lib, data, seg=0, stats=None):
    """the host chain over decode_block: what the device pass does, one block at a time"""
    out, pos, streams = bytearray(), 0, 0
    st = stats if stats is not None else {}
    st.update(blocks=0, trailing=0)
    while pos < len(data):
        hdr = data[pos: pos + 4]
        if not (hdr[:3] == b"BZh"[:len(hdr[:3])] and (len(hdr) < 4 or 0x31 <= hdr[3] <= 0x39)):
            if streams:
                st["trailing"] = len(data) - pos
                break
            raise BzError("not bzip2")
        if len(hdr) < 4:
            raise BzError("truncated header")
        level = hdr[3] - 0x30
        bit, comb = (pos + 4) * 8, 0
        while True:
            if bit + 48 > len(data) * 8:
                raise BzError("truncated")
            m = bits_at(data, bit, 48)
            if m == ub.MAGIC_EOS:
                if bit + 80 > len(data) * 8:
                    raise BzError("truncated")
                if bits_at(data, bit + 48, 32) != comb:
                    raise BzError("stream crc")
                pos = (bit + 80 + 7) // 8
                streams += 1
                break
            r, L = decode_block(lib, data, bit)
            if r["status"] < 0:
                raise BzError(r["status"])
            if r["n"] > level * 100000:
                raise BzError(E_SIZE)
            o, crc = block_output(lib, L, r["orig_ptr"], seg)
            if o is None:
                raise BzError(E_RLE)
            if crc != r["crc"]:
                raise BzError("block crc")
            comb = (((comb << 1) | (comb >> 31)) & 0xFFFFFFFF) ^ crc
            out += o
            st["blocks"] += 1
            bit = r["end_bit"]
    st["streams"] = streams
    return bytes(out)


def fastq(n, seed, lo=60, hi=160):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi))
        seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, L)].tobytes()
        out.append(b"@r%d\n%s\n+\n%s\n" % (i, seq, rng.integers(35, 74, L, dtype=np.uint8).tobytes()))
    return b"".join(out)


def fasta(n, seed):
    rng = np.random.default_rng(seed)
    return b"".join(b">s%d\n%s\n" % (i, np.frombuffer(b"ACGTN", dtype=np.uint8)[rng.integers(0, 5, int(rng.integers(20, 400)))].tobytes()) for i in range(n))


def payloads():
    rng = np.random.default_rng(1)
    runs = b"".join(bytes([65 + i % 20]) * k + b"x" for i, k in enumerate((3, 4, 5, 259, 260, 1000, 4, 3, 8, 255, 256, 257, 258)))
    return {
        "fastq": fastq(3000, 1),
        "fasta": fasta(1500, 2),
        "random": rng.integers(0, 256, 200000, dtype=np.uint8).tobytes(),
        "all_bytes": bytes(range(256)) * 7,
        "one_byte": b"Q",
        "runs": runs,
        "periodic_ab": b"ab" * 50000,
        "periodic_record": b"@r\nACGTACGTTT\n+\nFFFFFFFFFF\n" * 4000,
        "zeros": bytes(300000),
    }


@pytest.mark.parametrize("name", list(payloads()))
def test_payloads_match_bz2(bz, name):
    data = payloads()[name]
    for level in (1, 9):
        comp = bz2.compress(data, level)
        assert decompress(bz, comp) == data, (name, level)
    assert decompress(bz, bz2.compress(data, 5), seg=4096) == data
    assert decompress(bz, bz2.compress(data, 5), seg=7) == data


def test_every_level_and_concatenated_and_empty_streams(bz):
    data = fastq(6000, 3)
    for level in range(1, 10):
        comp = bz2.compress(data, level)
        st = {}
        assert decompress(bz, comp, stats=st) == data, level
        assert st["blocks"] == -(-len(ub.rle1(data)) // (level * 100000)) or level == 1, (level, st)
    empty = bz2.compress(b"")
    assert decompress(bz, empty) == b""
    parts = [bz2.compress(data[:5000], 1), empty, bz2.compress(data, 9), empty, bz2.compress(b"x", 3)]
    st = {}
    assert decompress(bz, b"".join(parts), stats=st) == data[:5000] + data + b"x"
    assert st["streams"] == 5
    st = {}
    assert decompress(bz, bz2.compress(data) + b"\0\0garbage", stats=st) == data and st["trailing"] == 9


def test_each_ngroups_and_a_full_random_block(bz):
    rng = np.random.default_rng(4)
    seen = set()
    for n in (20, 150, 400, 1000, 1800, 8000):            # nGroups follows the number of MTF symbols: < 200, 600, 1200, 2400
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        comp = bz2.compress(data)
        r, _ = decode_block(bz, comp, 32)
        seen.add(r["n_groups"])
        assert decompress(bz, comp) == data
    assert seen == {2, 3, 4, 5, 6}, seen
    data = rng.integers(0, 256, 899000, dtype=np.uint8).tobytes()
    comp = bz2.compress(data, 9)
    r, _ = decode_block(bz, comp, 32)
    assert r["status"] == 0 and r["n"] >= 899000 and r["n_selectors"] > 17000
    assert decompress(bz, comp, seg=4096) == data


def test_crc_combine_matches_a_direct_crc(bz):
    rng = np.random.default_rng(5)
    data = rng.integers(0, 256, 5000, dtype=np.uint8).tobytes()
    assert bz.bzh_crc(data, len(data)) == ub.crc32(data)
    for seg in (1, 3, 64, 4096):
        L, orig = ub.bwt(ub.rle1(data))
        o, crc = block_output(bz, np.frombuffer(L, dtype=np.uint8), orig, seg)
        assert o == data and crc == ub.crc32(data)


def test_truncations_and_bit_flips(bz):
    data = fastq(1500, 6)
    comp = bz2.compress(data, 1) + bz2.compress(data[:3000], 2)
    for cut in sorted(set([1, 3, 4, 5, 9, 10, 20, len(comp) - 1, len(comp) - 5, len(comp) - 10]) | set(range(30, len(comp) - 1, 1013))):
        with pytest.raises(BzError):
            decompress(bz, comp[:cut])
    rng = np.random.default_rng(7)
    errors = 0
    for t in range(200):
        b = bytearray(comp)
        i = int(rng.integers(4, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
        try:
            got = decompress(bz, bytes(b))
            assert got == data + data[:3000]
        except BzError:
            errors += 1
    assert errors > 190


def crafted(n_groups=2, **kw):
    data = fastq(40, 8)
    L, orig = ub.bwt(ub.rle1(data))
    syms, used = ub.mtf_symbols(L)
    blk = dict(syms=syms, used=used, orig_ptr=orig, out=data, n_groups=n_groups)
    blk.update(kw)
    return data, ub.stream([blk])


def test_writer_round_trips_through_bz2():
    for data in (fastq(50, 9), b"ab" * 300, bytes(1000), b"z"):
        assert bz2.decompress(ub.stream([data])) == data
    data, comp = crafted(n_groups=6, selectors=None)
    assert bz2.decompress(comp) == data


def crafted_status(bz, comp):
    r, _ = decode_block(bz, comp, 32)
    return r["status"]


def test_crafted_malformed_blocks(bz):
    data, good = crafted()
    assert crafted_status(bz, good) == 0 and decompress(bz, good) == data
    assert crafted_status(bz, crafted(randomised=1)[1]) == E_RANDOMISED
    n = len(ub.unrle1(ub.rle1(data)))
    _, comp = crafted(orig_ptr=len(ub.rle1(data)))
    assert crafted_status(bz, comp) == E_ORIGPTR
    with pytest.raises(OSError):
        bz2.decompress(comp)
    assert n == len(data)
    assert crafted_status(bz, crafted(start_len=0)[1]) == E_LENGTHS
    assert crafted_status(bz, crafted(start_len=21)[1]) == E_LENGTHS
    assert crafted_status(bz, crafted(n_groups=2, selectors=[0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0])[1]) == E_SELECTORS
    assert crafted_status(bz, crafted(n_selectors=0)[1]) == E_SELECTORS
    assert crafted_status(bz, crafted(n_groups=1)[1]) == E_GROUPS
    assert crafted_status(bz, crafted(n_groups=7)[1]) == E_GROUPS
    # selectors past 18 002 are read and ignored (libbz2 1.0.8)
    data2, many = crafted(extra_selectors=20000)
    assert bz2.decompress(many) == data2 and decompress(bz, many) == data2
    # numInUse = 0: an empty symbol map
    w = ub.BitWriter()
    w.put(int.from_bytes(b"BZh9", "big"), 32)
    w.put(ub.MAGIC_BLOCK, 48); w.put(0, 32); w.put(0, 1); w.put(0, 24); w.put(0, 16); w.put(0, 64)
    assert crafted_status(bz, w.bytes()) == E_MAP
    with pytest.raises(OSError):
        bz2.decompress(w.bytes())


def magic_block(seed=0):
    """a block whose coded data spells the block magic: 14 bytes in use, every symbol a 4-bit code, so the symbols
    3 1 4 1 5 9 2 6 5 3 5 9 are the magic's nibbles.  Filler symbols around them are drawn until the LF permutation
    is a single cycle (a block an encoder could have written)."""
    used = list(b"ABCDEFGHIJKLMN")
    spell = [3, 1, 4, 1, 5, 9, 2, 6, 5, 3, 5, 9]
    rng = np.random.default_rng(seed)
    for _ in range(2000):
        head = [int(x) for x in rng.integers(2, 15, 37)]
        tail = [int(x) for x in rng.integers(2, 15, 40)]
        syms = head + spell + tail + [15]
        L = ub.unmtf(syms, used)
        if ub.lf_cycles(L) != 1:
            continue
        for orig in range(len(L)):
            D = ub.unbwt(L, orig)
            try:
                out = ub.unrle1(D)
            except AssertionError:
                continue
            return dict(syms=syms, used=used, orig_ptr=orig, out=out, lengths=[4] * 16), out
    raise AssertionError("no single-cycle filler found")


def test_block_magic_inside_coded_data(bz):
    blk, out = magic_block()
    comp = ub.stream([blk])
    assert bz2.decompress(comp) == out
    assert decompress(bz, comp) == out
    found = scan(bz, comp)
    starts = [b for b in found if b >= 0]
    assert 32 in starts and len(starts) >= 2, found      # the real start and the false one inside the data
    real_end = decode_block(bz, comp, 32)[0]["end_bit"]
    for b in starts[1:]:
        assert 32 < b < real_end
        r, _ = decode_block(bz, comp, b)                  # decoding from the false start ends cleanly
        assert r["status"] < 0 or r["end_bit"] <= len(comp) * 8


def test_code_length_steps_are_capped(bz):
    """an encoder writes at most 19 +1/-1 steps per code length; a block that pads them is an error at once instead of
    reading through the whole input (every block the decoder accepts then fits in a bounded look-ahead)"""
    comp = ub.padded_lengths_stream(1 << 20)
    r, _ = decode_block(bz, comp, 32)
    assert r["status"] == E_LENGTHS, r
    data, padded = crafted(pad_steps=20)    # 40 steps to one length: accepted, as libbz2 does
    assert bz2.decompress(padded) == data and decompress(bz, padded) == data
    _, over = crafted(pad_steps=21)         # 42 steps: libbz2 reads on, this decoder stops
    assert bz2.decompress(over) == data and crafted_status(bz, over) == E_LENGTHS
