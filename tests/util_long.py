"""Long units (a mate longer than 60 000 bases) on the adversarial genomes: read sets for the device grid
(test_gpu_long_unit_grid.py) and read files for centrifuge-class and the oracle's file driver (test_long_unit_files.py).

The reads come from write_adversarial(seed=33), the genomes of the committed adv* indexes: sequence 0 and its reverse complement
(sequence 1), a 2 % mutant of sequence 0 (2) and of part of its reverse complement (3), a 5 600-base period-7 tandem repeat (4),
3 000-base A and T runs (5), a 150-base repeat in 300 copies (6, 105 000 bases, the only sequence over 65 550 bases), a 30-copy
repeat (7) and 12 random 4 kb sequences.  A long strand is searched in segments of SEG bases counted in search positions: the
forward strand's position p is read offset len - 1 - p, the reverse strand's is p."""
import atexit
import functools
import json
import os

import numpy as np

import util

LONG = 60000                      # kLongUnitLen: a unit with a longer mate takes the segmented path
SEG = 4096                        # kSegLen: bases per speculative chain
FTAB_CHARS = {"adv": 10, "adv_t1o2": 1, "adv_t6o0": 6, "adv_t8o7": 8}


@functools.lru_cache(None)
def genomes():
    """the adv genomes as codes 0..3"""
    d = os.path.join(util.CACHE, "adv_genomes")
    if not os.path.exists(os.path.join(d, "genomes.fa")):
        util.synth.write_adversarial(d, seed=33, n_reads=10)
    return [util.ASC2DNA[a] & 3 for _, a in util.parse_reads(os.path.join(d, "genomes.fa"))]


def kmer_k(name):
    """K of the index's K-mer table as the loader picks it: from ftabChars up while K < 15 and 4^(K+1) <= len/4"""
    k, n = FTAB_CHARS[name], sum(len(s) for s in genomes())
    while k < 15 and 4 ** (k + 1) <= n // 4:
        k += 1
    return k


def rc(codes):
    return (3 - codes)[::-1]


def ascii_(codes, rng=None, sub=0.0):
    """codes -> ASCII bases, with a fraction `sub` of them substituted"""
    r = np.array(codes, dtype=np.uint8)
    if sub:
        m = rng.random(len(r)) < sub
        r[m] = (r[m] + 1 + rng.integers(0, 3, size=int(m.sum()), dtype=np.uint8)) & 3
    return util.synth.ACGT[r].copy()


def revcomp(a):
    return np.frombuffer(a.tobytes()[::-1].translate(bytes.maketrans(b"ACGTN", b"TGCAN")), dtype=np.uint8).copy()


def with_ns(a, frac, rng):
    a = a.copy()
    a[rng.random(len(a)) < frac] = ord("N")
    return a


def chimera(length, rng, sub=0.01):
    """pieces of several sequences from both strands"""
    seqs, out, have = genomes(), [], 0
    while have < length:
        s = seqs[int(rng.integers(len(seqs)))]
        n = min(int(rng.integers(1500, 30000)), len(s), length - have)
        p = int(rng.integers(0, len(s) - n + 1))
        piece = s[p:p + n]
        out.append(rc(piece) if rng.random() < 0.5 else piece)
        have += n
    return ascii_(np.concatenate(out), rng, sub)


def search_pos_ns(a, positions):
    """Ns at these search positions on both strands: read offsets p (reverse strand) and len - 1 - p (forward strand)"""
    a = a.copy()
    for p in positions:
        a[p] = a[len(a) - 1 - p] = ord("N")
    return a


def with_islands(a):
    """Exact A and T runs of 2 986 - 2 990 bases between two Ns: both strands' chains stop at the Ns, so each run is one hit
    on either strand over the same bases.  The index holds one 3 000-base A run and one T run, so each hit is 11 - 15 SA rows
    wide (scored: at most ihits = 20) and the pair is wider than ihits: twins that twin removal clears."""
    parts, p = [], 0
    for q, run in ((4000, b"A" * 2986), (30000, b"T" * 2990), (60000, b"T" * 2986)):
        parts += [a[p:q], np.frombuffer(b"N" + run + b"N", dtype=np.uint8)]
        p = q
    return np.concatenate(parts + [a[p:]])


@functools.lru_cache(None)
def long_reads(k):
    """The long reads of the grid, by name; `k` is the K-mer table's K the boundary Ns are placed for."""
    s = genomes()
    rng = np.random.default_rng(61)
    r = {}
    r["s0_s1"] = ascii_(np.concatenate([s[0][10000:], s[1][:50000]]), rng, 0.01)             # every hit has a partner on the other strand
    r["repeats"] = with_islands(ascii_(np.concatenate([s[4], s[5], s[6][:40000], rc(s[4]), rc(s[5]), s[7]]), rng, 0.01))    # tandem, A/T runs, dispersed
    r["chimera"] = chimera(90000, rng)
    r["exact70k"] = ascii_(s[6][20000:90000])                  # one hit of 70 000 bases: (len - 15)^2 wraps in 32 bits
    cut = ascii_(s[6][1000:62000], rng, 0.01)
    r["cut60000"], r["cut60001"] = cut[:LONG], cut[:LONG + 1]  # the short path through k_search_long, and the long path
    edge = chimera(16 * SEG + 2, rng)
    for d in (-1, 0, 1):
        r["edge%+d" % d] = edge[:15 * SEG + d]                   # the last segment full, one base short of it, or a single base
    b = [SEG * i for i in range(1, 16)]
    r["edge_ns"] = search_pos_ns(edge[:16 * SEG + 2], [b[0] - 1, b[2], b[4] - 1, b[4], b[6] + k - 1, b[8] + k, b[10] + 1]
                                 + list(range(b[12] - 20, b[12] + 21)))   # last / first base of a segment, the first K-mer, a run across
    return r


def short_reads(n, seed):
    return [a for _, a in util.synth.sample_reads(genomes(), n, 150, seed=seed, lens=(20, 400))]


def place(longs, shorts, at):
    """shorts with longs[i] inserted so that it ends up at unit index at[i]"""
    out = list(shorts)
    for i, a in sorted(zip(at, range(len(longs)))):
        out.insert(i, longs[a])
    return out


SE_AT = [0, 31, 32, 63, 64, 95, 96, 120, 127, 128, 150]        # warp boundaries of the per-unit stages


@functools.lru_cache(None)
def single_set(k):
    """(mates, names of the long units) of the single-end batch"""
    lr = long_reads(k)
    names = ["s0_s1", "repeats", "chimera", "exact70k", "cut60000", "cut60001", "edge-1", "edge+0", "edge+1", "edge_ns"]
    longs = [lr[x] for x in names] + [with_ns(lr["chimera"][:61000], 0.2, np.random.default_rng(3))]    # fails the N filter
    reads = place(longs, short_reads(160, 71), SE_AT)
    return reads, names + ["nfail"]


PE_SHAPES = ["twins_repeats", "twins_s0_s1", "unrelated", "long_short", "short_long", "long_empty", "nfail_pass", "pass_nfail",
             "long_nfail", "both_fail", "edges", "edge_ns_short"]


@functools.lru_cache(None)
def pair_units(k):
    """the long pairs of the paired batch, by shape: (mate 1, mate 2)"""
    lr = long_reads(k)
    rng = np.random.default_rng(62)
    sh = short_reads(8, 72)
    nf = with_ns(chimera(65000, rng), 0.2, rng)
    u = {"twins_repeats": (lr["repeats"], revcomp(lr["repeats"])), "twins_s0_s1": (lr["s0_s1"], revcomp(lr["s0_s1"])),
         "unrelated": (lr["chimera"], lr["exact70k"]), "long_short": (lr["cut60001"], sh[0]), "short_long": (sh[1], lr["edge+1"]),
         "long_empty": (lr["edge+0"], np.zeros(0, dtype=np.uint8)), "nfail_pass": (nf, sh[2]), "pass_nfail": (sh[3], nf),
         "long_nfail": (lr["chimera"], nf), "both_fail": (nf, with_ns(sh[4], 0.5, rng)), "edges": (lr["edge-1"], lr["edge+1"]),
         "edge_ns_short": (lr["edge_ns"], lr["cut60000"])}
    return u


def replaced_twins(k):
    """the twin pairs with mate 2 replaced by an unrelated long read"""
    u, other = pair_units(k), chimera(70000, np.random.default_rng(63))
    return {x: (u[x][0], other) for x in ("twins_repeats", "twins_s0_s1")}


PE_AT = [0, 31, 32, 33, 63, 64, 90, 95, 96, 127, 128, 140]


def pair_batch_of(units):
    s1, s2 = short_reads(130, 73), short_reads(130, 74)
    shorts = list(zip(s1, s2))
    pairs = place([units[x] for x in PE_SHAPES], shorts, PE_AT)
    return [x for x, _ in pairs], [y for _, y in pairs]


@functools.lru_cache(None)
def pair_set(k):
    return pair_batch_of(pair_units(k))


def long_units_of(mates1, mates2=None):
    """number of units the segmented path takes: a mate longer than LONG bases"""
    return sum(1 for i in range(len(mates1)) if len(mates1[i]) > LONG or (mates2 is not None and len(mates2[i]) > LONG))


# ------------------------------------------------------------------------------ read files for centrifuge-class
THRESH = (LONG - 1, LONG, LONG + 1, LONG + 10)
TRIMS = [(0, 0), (0, 1), (1, 0), (10, 0), (0, 11), (5, 6), (0, 2)]


def cli_read_files(d=None):
    """FASTQ and FASTA files in d (None: none written): single, paired with long twins and long mates that fail the N filter,
    and the threshold reads of THRESH bases.  Returns the (name, read) lists: {se, pe: (mates 1, mates 2), th, th_pe}."""
    lr = long_reads(kmer_k("adv"))
    rng = np.random.default_rng(64)
    se = [("s%d" % i, a) for i, a in enumerate(short_reads(60, 81))]
    for i, x in enumerate(["s0_s1", "repeats", "exact70k", "cut60000", "cut60001", "edge_ns"]):
        se.insert(5 + 9 * i, ("l_" + x, lr[x]))
    se.insert(40, ("l_nfail", with_ns(lr["chimera"][:62000], 0.2, rng)))
    m1 = [("p%d" % i, a) for i, a in enumerate(short_reads(40, 82))]
    m2 = [(n, revcomp(a)) for n, a in m1]
    nf = with_ns(lr["chimera"][:64000], 0.2, rng)
    longs = [("tw_rep", lr["repeats"], revcomp(lr["repeats"])), ("tw_s0", lr["s0_s1"], revcomp(lr["s0_s1"])),
             ("lnf", lr["chimera"], nf), ("nfs", nf, m1[0][1]), ("snf", m1[1][1], nf), ("lsh", lr["cut60001"], m1[2][1])]
    for i, (n, a, b) in enumerate(longs):
        m1.insert(3 + 6 * i, (n, a)); m2.insert(3 + 6 * i, (n, b))
    cut = ascii_(genomes()[6][30000:30000 + LONG + 10], rng, 0.01)
    th = [("s%d" % i, a) for i, a in enumerate(short_reads(30, 83))]
    for i, n in enumerate(THRESH):
        th.insert(4 + 7 * i, ("t%d" % n, cut[:n]))
    th2 = [(n, revcomp(a) if len(a) > 1000 else a[::-1].copy()) for n, a in th]
    for tag, reads in (("se", se), ("p_1", m1), ("p_2", m2), ("th", th), ("th_2", th2)):
        for fmt in ("fq", "fa") if d else ():
            p = os.path.join(d, "%s.%s" % (tag, fmt))
            (util.synth.write_fastq if fmt == "fq" else util.synth.write_fasta)(p, reads)
    return {"se": se, "pe": (m1, m2), "th": th, "th_pe": (th, th2)}


def cli_cases(d=None, base=""):
    """(key, centrifuge-class arguments, units, long units implied by the trimmed lengths) of every file case, on the files
    cli_read_files writes in d"""
    reads = cli_read_files(d)
    d = d or ""
    out = []
    for fmt, flag in (("fq", "-q"), ("fa", "-f")):
        f = lambda t: os.path.join(d, "%s.%s" % (t, fmt))       # noqa: E731
        out.append(("se_" + fmt, [flag, "-x", base, "-U", f("se")], reads["se"], None))
        out.append(("pe_" + fmt, [flag, "-x", base, "-1", f("p_1"), "-2", f("p_2")], *reads["pe"]))
    for t5, t3 in TRIMS:
        tr = ["--trim5", str(t5), "--trim3", str(t3)]
        out.append(("th_%d_%d" % (t5, t3), ["-q", "-x", base, "-U", os.path.join(d, "th.fq")] + tr, reads["th"], None))
        if (t5, t3) in ((0, 0), (0, 1), (10, 0)):
            out.append(("th_pe_%d_%d" % (t5, t3), ["-f", "-x", base, "-1", os.path.join(d, "th.fa"), "-2", os.path.join(d, "th_2.fa")] + tr,
                        *reads["th_pe"]))
    cases = []
    for key, args, m1, m2 in out:
        t5 = int(args[args.index("--trim5") + 1]) if "--trim5" in args else 0
        t3 = int(args[args.index("--trim3") + 1]) if "--trim3" in args else 0
        tl = lambda n: max(0, n - t5 - t3)                       # noqa: E731
        n_long = sum(1 for i in range(len(m1)) if tl(len(m1[i][1])) > LONG or (m2 is not None and tl(len(m2[i][1])) > LONG))
        cases.append((key, args, len(m1), n_long))
    return cases


DIGESTS = os.path.join(util.GOLDEN, "long_unit_digests.json")
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
    if util.RECORD:
        if not util.have_ref():
            raise RuntimeError("CFB_RECORD_REFERENCE=1 needs the reference binaries under oracle/_ref (make -C oracle ref)")
        if not _recorded:
            atexit.register(_save_digests)
        _recorded[key] = util.digest(util.run_cli(util.REF_CLASS, args, os.path.join(str(tmp), "ref.tsv"), os.path.join(str(tmp), "ref.rep")))
        return _recorded[key]
    with open(DIGESTS) as f:
        digests = json.load(f)
    if key not in digests:
        raise KeyError("no recorded reference output for %r (re-record with CFB_RECORD_REFERENCE=1)" % key)
    return digests[key]
