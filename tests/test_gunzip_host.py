"""The device inflater's per-chunk decoder (centrifuge_b200/csrc/cf_inflate.h), compiled for the host by
tests/native/gunzip_host.cpp and checked against zlib: every block type and zlib strategy, flush points, decoding from
every block boundary with the window unknown (markers) and then resolved from the true window, the block-start search
on real and false starts, and malformed streams, which must end in an error status within the bounds of the input."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import util

NONE = (1 << 64) - 1
ST_STOP, ST_END, ST_FULL = 1, 2, 3
E_INPUT, E_BTYPE, E_STORED, E_CODES, E_SYM = -1, -2, -3, -4, -5
WIN = 32768


@pytest.fixture(scope="module")
def gz(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("gunzip_host") / "gunzip_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(util.ROOT, "tests", "native", "gunzip_host.cpp")])
    lib = C.CDLL(so)
    lib.gzh_scan.restype = C.c_uint64
    return lib


def chunk(lib, comp, start_bit=0, stop_bit=NONE, start_hdr=NONE, cap=None):
    """decode comp from a state: (result dict, symbols)"""
    buf = np.frombuffer(comp, dtype=np.uint8) if len(comp) else np.zeros(1, dtype=np.uint8)
    cap = cap if cap is not None else max(1024, len(comp) * 1100 + 1024)
    out = np.zeros(cap, dtype=np.uint16)
    res = np.zeros(8, dtype=np.int64)
    lib.gzh_inflate_chunk(buf.ctypes.data_as(C.c_void_p), C.c_uint64(len(comp)), C.c_uint64(start_bit), C.c_uint64(start_hdr),
                          C.c_uint64(stop_bit), out.ctypes.data_as(C.c_void_p), C.c_uint32(cap), res.ctypes.data_as(C.c_void_p))
    r = dict(zip(("status", "n_sym", "end_bit", "end_hdr", "safe_bit", "safe_hdr", "safe_sym", "first_type"), (int(x) for x in res)))
    for k in ("end_hdr", "safe_hdr"):
        r[k] &= NONE
    assert 0 <= r["n_sym"] <= cap
    return r, out[: r["n_sym"]]


def scan(lib, comp, lo, hi, verified=False):
    buf = np.frombuffer(comp, dtype=np.uint8)
    out = np.zeros(max(1, hi - lo), dtype=np.uint64)
    k = lib.gzh_scan(buf.ctypes.data_as(C.c_void_p), C.c_uint64(len(comp)), C.c_uint64(lo), C.c_uint64(hi), out.ctypes.data_as(C.c_void_p),
                     C.c_uint64(len(out)), C.c_int(1 if verified else 0))
    return set(int(x) for x in out[:k])


def resolve(syms, window):
    """markers -> bytes of the 32 KB window before the chunk (window: the true preceding bytes, any length)"""
    w = np.zeros(WIN, dtype=np.uint8)
    tail = np.frombuffer(window[-WIN:], dtype=np.uint8)
    w[WIN - len(tail):] = tail
    m = syms >= 256
    assert not m.any() or int((syms[m] - 256).min()) >= WIN - len(tail), "marker before the start of the output"
    out = syms.astype(np.uint8)
    out[m] = w[syms[m] - 256]
    return out.tobytes()


def raw(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=(), zdict=None):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy, **({"zdict": zdict} if zdict else {}))
    parts, pos = [], 0
    for at, mode in flushes:
        parts += [c.compress(data[pos:at]), c.flush(mode)]
        pos = at
    parts += [c.compress(data[pos:]), c.flush()]
    return b"".join(parts)


def fastq(n, seed, lo=60, hi=160):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.integers(lo, hi))
        seq = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, L)].tobytes()
        q = rng.integers(35, 74, L, dtype=np.uint8).tobytes()
        out.append(b"@read_%d/1\n%s\n+\n%s\n" % (i, seq, q))
    return b"".join(out)


def mixed(seed):
    rng = np.random.default_rng(seed)
    return fastq(3000, seed) + rng.integers(0, 256, 40000, dtype=np.uint8).tobytes() + b"ACGT" * 30000 + bytes(70000) + fastq(1500, seed + 1)


def boundaries(lib, comp):
    """[(bit, output offset)] of every block start, found by decoding one block at a time from the stream start"""
    out, bit, off = [], 0, 0
    while True:
        out.append((bit, off))
        r, syms = chunk(lib, comp, bit, bit + 1)
        assert r["status"] in (ST_STOP, ST_END), r
        off += r["n_sym"]
        if r["status"] == ST_END:
            return out, off, r["end_bit"]
        bit = r["end_bit"]


CASES = ([("level%d" % lv, dict(level=lv)) for lv in (0, 1, 6, 9)]
         + [(n, dict(strategy=getattr(zlib, n))) for n in ("Z_FILTERED", "Z_HUFFMAN_ONLY", "Z_RLE", "Z_FIXED")]
         + [("sync_flush", dict(flushes=[(50000, zlib.Z_SYNC_FLUSH), (50001, zlib.Z_SYNC_FLUSH), (300000, zlib.Z_SYNC_FLUSH)])),
            ("full_flush", dict(flushes=[(70000, zlib.Z_FULL_FLUSH), (400000, zlib.Z_FULL_FLUSH)]))])


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_every_block_boundary_decodes_to_zlib(gz, name, kw):
    data = mixed(len(name))
    comp = raw(data, **kw)
    r, syms = chunk(gz, comp)
    assert r["status"] == ST_END and syms.astype(np.uint8).tobytes() == data and (syms < 256).all()
    assert r["end_bit"] <= len(comp) * 8 and (r["end_bit"] + 7) // 8 == len(comp)
    bds, total, _ = boundaries(gz, comp)
    assert total == len(data) and len(bds) > 2
    found = scan(gz, comp, 0, len(comp) * 8)
    verified = scan(gz, comp, 0, len(comp) * 8, verified=True)
    assert verified <= found
    for i, (bit, off) in enumerate(bds):
        # unknown window: markers, resolved from the true preceding bytes, give zlib's bytes up to the next boundary
        nxt = bds[i + 1][1] if i + 1 < len(bds) else total
        r, syms = chunk(gz, comp, bit, bit + 1)
        assert r["n_sym"] == nxt - off
        assert resolve(syms, data[:off]) == data[off:nxt], (name, i)
        # block starts the search is meant to find: dynamic blocks and non-final stored blocks
        if r["first_type"] == 2 or (r["first_type"] == 0 and r["status"] != ST_END):
            assert bit in found and bit in verified, (name, i, r)
    # a few long decodes from the middle, across many blocks
    for bit, off in bds[1::max(1, len(bds) // 4)]:
        r, syms = chunk(gz, comp, bit)
        assert r["status"] == ST_END and resolve(syms, data[:off]) == data[off:]


def test_known_window_from_a_preset_dictionary(gz):
    """A raw stream compressed against a dictionary refers to it from its first block: markers name its bytes."""
    zd = fastq(400, 9)
    data = fastq(2000, 9)[5000:]
    comp = raw(data, zdict=zd)
    r, syms = chunk(gz, comp)
    assert r["status"] == ST_END and (syms >= 256).any()
    assert resolve(syms, zd) == data


def test_false_starts_do_not_crash_and_are_rare(gz):
    rng = np.random.default_rng(3)
    data = fastq(4000, 3)
    comp = raw(data)
    bds, _, _ = boundaries(gz, comp)
    real = set(b for b, _ in bds)
    found = scan(gz, comp, 0, len(comp) * 8)
    false = sorted(found - real)
    assert len(false) < len(comp) * 8 // 2000, len(false)
    assert len(scan(gz, comp, 0, len(comp) * 8, verified=True) - real) <= len(false) // 20
    for b in false:                            # decoding from a false start must end cleanly, whatever it produces
        r, _ = chunk(gz, comp, b, cap=1 << 20)
        assert r["status"] in (ST_STOP, ST_END, ST_FULL) or r["status"] < 0
    noise = rng.integers(0, 256, 200000, dtype=np.uint8).tobytes()
    for b in sorted(scan(gz, noise, 0, len(noise) * 8))[:200]:
        r, _ = chunk(gz, noise, b, cap=1 << 20)
        assert r["end_bit"] <= len(noise) * 8 + 64


def test_full_buffer_resumes_mid_block(gz):
    data = bytes(3_000_000) + fastq(3000, 4)
    comp = raw(data, level=9)
    got, bit, hdr, pieces = b"", 0, NONE, 0
    for pieces in range(1, 10000):
        r, syms = chunk(gz, comp, bit, start_hdr=hdr, cap=100000)
        got += resolve(syms, got)
        if r["status"] == ST_END:
            break
        assert r["status"] == ST_FULL, r
        bit, hdr = r["end_bit"], r["end_hdr"]
    assert got == data and pieces > 30


def test_malformed_streams_end_in_an_error(gz):
    data = fastq(800, 5)
    comp = raw(data)
    for k in list(range(0, 64)) + list(range(64, len(comp) - 1, 97)):
        r, _ = chunk(gz, comp[:k])
        assert r["status"] == E_INPUT or (r["status"] < 0), (k, r)
    rng = np.random.default_rng(6)
    for t in range(300):
        b = bytearray(comp)
        for _ in range(1 + t % 3):
            i = int(rng.integers(0, len(b)))
            b[i] ^= 1 << int(rng.integers(0, 8))
        r, syms = chunk(gz, bytes(b), cap=len(data) * 2)
        assert r["end_bit"] <= len(b) * 8 + 64
        if r["status"] == ST_END and syms.astype(np.uint8).tobytes() != data:
            pass                               # wrong bytes from a valid-looking stream: the gzip CRC-32 rejects them
    pad = bytes(16)                            # errors within a code's reach of the end of the input count as running out of it
    assert chunk(gz, b"\x07" + pad)[0]["status"] == E_BTYPE                                  # BFINAL 1, BTYPE 3
    assert chunk(gz, b"\x07")[0]["status"] == E_INPUT
    assert chunk(gz, b"\x01\x05\x00\xfb\xff" + b"x" * 5 + pad)[0]["status"] == E_STORED      # NLEN != ~LEN
    assert chunk(gz, b"\x01\x05\x00\xfa\xff" + b"x" * 4)[0]["status"] == E_INPUT            # stored data cut short
    assert chunk(gz, bytes([0x05 | (30 << 3), 0xff, 0xff]) + pad)[0]["status"] == E_CODES    # HLIT = 287
    # fixed block: literal/length code 286 (11000110, 8 bits) is invalid
    bits = [1, 1, 0] + [1, 1, 0, 0, 0, 1, 1, 0]
    v = sum(b << i for i, b in enumerate(bits))
    assert chunk(gz, v.to_bytes(2, "little") + pad)[0]["status"] == E_SYM
    r, _ = chunk(gz, b"")
    assert r["status"] == E_INPUT
