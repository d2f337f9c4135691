"""A small bzip2 writer for crafted streams: rotation sort, RLE1, MTF/RLE2, canonical Huffman codes with explicit or
computed lengths, selectors, and the stream and block headers.  Its output decodes with Python's bz2; the tests use it
to write blocks that no encoder writes on its own (bad fields, a block magic inside a block's coded data)."""
import heapq

MAGIC_BLOCK = 0x314159265359
MAGIC_EOS = 0x177245385090


def crc32(data):
    """bzip2's CRC-32: polynomial 0x04C11DB7, MSB first, init and final xor 0xFFFFFFFF"""
    c = 0xFFFFFFFF
    for b in data:
        c ^= b << 24
        for _ in range(8):
            c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
    return c ^ 0xFFFFFFFF


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

    def tell(self):
        return len(self.bits)

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(int("".join(map(str, b[i:i + 8])), 2) for i in range(0, len(b), 8))


def rle1(data):
    out, i = bytearray(), 0
    while i < len(data):
        j = i
        while j < len(data) and data[j] == data[i] and j - i < 255 + 4:
            j += 1
        k = j - i
        if k >= 4:
            out += bytes([data[i]]) * 4 + bytes([k - 4])
        else:
            out += data[i:j]
        i = j
    return bytes(out)


def unrle1(d):
    out, r, prev = bytearray(), 0, None
    for x in d:
        if r == 4:
            out += bytes([prev]) * x
            r = 0
        else:
            r = r + 1 if r > 0 and x == prev else 1
            out.append(x)
        prev = x
    assert r != 4, "ends after four equal bytes"
    return bytes(out)


def bwt(d):
    """(L, origPtr) by sorting the rotations of d (small blocks only: the sort keys are copies of every rotation)"""
    n = len(d)
    assert n <= 50000, "the test writer sorts rotations as whole copies"
    dd = d + d
    order = sorted(range(n), key=lambda i: dd[i:i + n])
    return bytes(d[(i - 1) % n] for i in order), order.index(0)


def unbwt(L, orig):
    """libbz2's walk: n steps from tt[origPtr] (repeating the cycle of a periodic block)"""
    n = len(L)
    order = sorted(range(n), key=lambda i: (L[i], i))
    p = order[orig]
    out = bytearray()
    for _ in range(n):
        out.append(L[p])
        p = order[p]
    return bytes(out)


def lf_cycles(L):
    n = len(L)
    order = sorted(range(n), key=lambda i: (L[i], i))
    seen, cycles = [False] * n, 0
    for s in range(n):
        if not seen[s]:
            cycles += 1
            while not seen[s]:
                seen[s] = True
                s = order[s]
    return cycles


def mtf_symbols(L):
    """(symbols, bytes in use) of the MTF/RLE2 stage, EOB last"""
    used = sorted(set(L))
    idx = {b: i for i, b in enumerate(used)}
    lst = list(range(len(used)))
    syms, z = [], 0

    def flush():
        nonlocal z
        if z:
            z -= 1
            while True:
                syms.append(z & 1)
                if z < 2:
                    break
                z = (z - 2) // 2
            z = 0
    for b in L:
        j = lst.index(idx[b])
        if j == 0:
            z += 1
            continue
        flush()
        syms.append(j + 1)
        lst.insert(0, lst.pop(j))
    flush()
    syms.append(len(used) + 1)
    return syms, used


def unmtf(syms, used):
    lst, out, run, w = list(range(len(used))), bytearray(), 0, 1
    for s in syms:
        if s <= 1:
            run += (s + 1) * w
            w <<= 1
            continue
        out += bytes([used[lst[0]]]) * run
        run, w = 0, 1
        if s == len(used) + 1:
            break
        j = s - 1
        lst.insert(0, lst.pop(j))
        out.append(used[lst[0]])
    return bytes(out)


def huffman_lengths(freq, maxlen=17):
    freq = [f + 1 for f in freq]
    while True:
        h = [(f, i, [i]) for i, f in enumerate(freq)]
        heapq.heapify(h)
        L = [0] * len(freq)
        k = len(freq)
        while len(h) > 1:
            f1, _, a = heapq.heappop(h)
            f2, _, b = heapq.heappop(h)
            for s in a + b:
                L[s] += 1
            heapq.heappush(h, (f1 + f2, k, a + b))
            k += 1
        if max(L) <= maxlen:
            return L
        freq = [1 + f // 2 for f in freq]


def codes(lengths):
    """canonical codes: in order of length, then symbol"""
    out, code = {}, 0
    for ln in range(1, 21):
        for s, x in enumerate(lengths):
            if x == ln:
                out[s] = code
                code += 1
        code <<= 1
    return out


def write_block(w, syms, used, orig_ptr, crc, n_groups=2, lengths=None, selectors=None, randomised=0, n_selectors=None,
                extra_selectors=0, start_len=None, pad_steps=0):
    """one block from its MTF/RLE2 symbols: every group gets `lengths` (else Huffman lengths of syms) unless lengths is
    a list of per-group lists; selectors default to 0 for every group of 50 symbols; pad_steps pairs of +1/-1 steps go
    before the first code length's own steps"""
    alpha = len(used) + 2
    if lengths is None:
        f = [0] * alpha
        for s in syms:
            f[s] += 1
        lengths = huffman_lengths(f)
    per_group = lengths if isinstance(lengths[0], (list, tuple)) else [lengths] * n_groups
    ngroups_sel = (len(syms) + 49) // 50
    if selectors is None:
        selectors = [0] * ngroups_sel
    selectors = list(selectors) + [0] * (max(0, ngroups_sel - len(selectors)) + extra_selectors)
    w.put(MAGIC_BLOCK, 48)
    w.put(crc, 32)
    w.put(randomised, 1)
    w.put(orig_ptr, 24)
    in16 = [any(b // 16 == i for b in used) for i in range(16)]
    w.put(sum(1 << (15 - i) for i in range(16) if in16[i]), 16)
    for i in range(16):
        if in16[i]:
            w.put(sum(1 << (15 - (b % 16)) for b in used if b // 16 == i), 16)
    w.put(n_groups, 3)
    w.put(len(selectors) if n_selectors is None else n_selectors, 15)
    order = list(range(max(n_groups, 6)))
    for s in selectors:
        j = order.index(s)
        w.put((1 << (j + 1)) - 2, j + 1)        # j ones, then a zero
        order.insert(0, order.pop(j))
    for t, ln in enumerate(per_group[:n_groups]):
        cur = ln[0] if start_len is None else start_len
        w.put(cur, 5)
        for _ in range(pad_steps if t == 0 else 0):
            w.put(0b10 if cur < 20 else 0b11, 2)
            w.put(0b11 if cur < 20 else 0b10, 2)
        for x in ln:
            while cur < x:
                w.put(0b10, 2)
                cur += 1
            while cur > x:
                w.put(0b11, 2)
                cur -= 1
            w.put(0, 1)
    tabs = [codes(ln) for ln in per_group[:n_groups]]
    for i, s in enumerate(syms):
        g = min(selectors[i // 50], len(tabs) - 1)        # (a selector past nGroups is an error before any symbol)
        w.put(tabs[g][s], per_group[g][s])


def stream(blocks, level=9):
    """blocks: raw byte strings, or dicts of write_block arguments plus 'out' (the block's output for the CRCs)"""
    w = BitWriter()
    w.put(int.from_bytes(b"BZh" + str(level).encode(), "big"), 32)
    comb = 0
    for b in blocks:
        if not isinstance(b, dict):
            L, orig = bwt(rle1(b))
            syms, used = mtf_symbols(L)
            b = dict(syms=syms, used=used, orig_ptr=orig, out=b)
        kw = dict(b)
        out = kw.pop("out")
        kw.setdefault("crc", crc32(out))
        comb = (((comb << 1) | (comb >> 31)) & 0xFFFFFFFF) ^ kw["crc"]
        write_block(w, **kw)
    w.put(MAGIC_EOS, 48)
    w.put(comb, 32)
    return w.bytes()


def padded_lengths_stream(pad_bytes, level=9):
    """a stream whose first block pads its first code length with pad_bytes * 4 pairs of +1/-1 steps ("10 11"): libbz2
    reads on through all of them, an encoder never writes more than 19 steps per length"""
    w = BitWriter()
    w.put(int.from_bytes(b"BZh" + str(level).encode(), "big"), 32)
    w.put(MAGIC_BLOCK, 48)
    w.put(0, 32)
    w.put(0, 1)
    w.put(0, 24)
    w.put(1 << 15, 16)                      # bytes 0..15 in use
    w.put(0xFFFF, 16)
    w.put(2, 3)
    w.put(1, 15)
    w.put(0, 1)                             # selector 0
    w.put(5, 5)                             # group 0 starts at length 5
    if w.tell() % 2:
        w.put(0b10110, 5)                   # symbol 0: +1, -1, stop (length 5)
    while w.tell() % 8:
        w.put(0b1011, 4) if w.tell() % 8 == 4 else w.put(0b10, 2)
    return w.bytes() + b"\xbb" * pad_bytes + bytes(64)
