"""Tie-rich fixture: genomes whose reads tie among an exact number of sequences, an NCBI-shaped taxonomy, dispersed repeats at
copy counts on both sides of the ihits thresholds, and reads and read files for the -k 1 to 64 grid.

Genomes (one seeded generator, about 0.55 Mbp):
  - seven genera of S = 2, 5, 16, 31, 32, 33 and 40 sequences.  Every sequence of a genus carries the genus's 1 000-base block,
    so a read from the block ties among exactly S sequences; the genera of family 10 also share a 400-base family block.
    Everything else is unique random sequence.
  - irregular lineages: a subgenus (genus 106), a subfamily and a tribe (genus 104), a species straight under family 11,
    strain, subspecies and "no rank" leaves under species (one beside a sequence of its species), a sequence mapped to its genus's taxid, a sequence whose taxid is
    missing from nodes.dmp, one missing from the conversion table, a node missing from names.dmp, and a "no rank" clade
    between family 10 and the root.  Taxids 10200 and 10300 have two sequences each.
  - dispersed repeats: one sequence per copy count (COPIES), each copy a 100-base unit of its own between random spacers.  A
    read from a unit hits one SA range of `copies` rows, which the classifier drops when it exceeds
    ihits = max(k, 5) x (4 with >= 10 `cid` names, else 40).
Two builds of the same genomes: "cid" (names cid<i>: ihits x 4) and "plain" (names seq<i>: ihits x 40).  That the fixture
reaches all this (every group size, a unit of more than 32 tied host records, every repeat moving at its threshold) is asserted
by tests/test_tie_grid_host.py.

The indexes are committed under tests/golden (ties_<build>.{1,2,3,4}.cf.xz): written by the reference builder when recording
(CFB_RECORD_REFERENCE=1), which also records their digests, against which the device tests check the project's own builder."""
import functools
import lzma
import os

import numpy as np

import util

A = util.synth.ACGT
SPECIES = (2, 5, 16, 31, 32, 33, 40)          # sequences per genus; genus g has taxid 100 + g
FAMILY_OF = {0: 10, 1: 10, 2: 10, 3: 10, 4: 11, 5: 11, 6: 11}
GENUS_BLOCK, FAMILY_BLOCK = 1000, 400
COPIES = (20, 21, 32, 33, 64, 65, 128, 129, 200, 201, 240, 241)
REPEAT_UNIT, REPEAT_GAP = 100, 40
BUILDS = ("cid", "plain")
HOST = (106, 10500, 10501, 10407)            # --host-taxids: the 40-sequence genus and three species
EXCL = (103, 10201)                          # --exclude-taxids: the 31-sequence genus and one species
K_GRID = (1, 2, 3, 4, 5, 6, 8, 15, 16, 17, 31, 32, 33, 40, 64)
LENGTHS = {"r128": (60, 128), "r160": (129, 160), "r320": (161, 320), "r900": (321, 900)}
MIXED_K = 32                                 # -k of the mixed file: every tie of genera 102-104 is a tie set


def ihits(build, k):
    return max(k, 5) * (4 if build == "cid" else 40)


def species_taxid(g, s):
    return 10000 + 100 * g + s


def seq_taxonomy():
    """[(taxid or None when missing from the conversion table)] per sequence, the nodes.dmp rows (taxid, parent, rank) and
    the taxids that get no names.dmp row"""
    nodes = [(1, 1, "no rank"), (5, 1, "no rank"), (10, 5, "family"), (11, 1, "family"), (12, 1, "family"),
             (20, 11, "subfamily"), (21, 20, "tribe"), (30, 106, "subgenus"), (190, 12, "genus")]
    tax = []
    for g, S in enumerate(SPECIES):
        nodes.append((100 + g, 21 if g == 4 else FAMILY_OF[g], "genus"))
        for s in range(S):
            t = species_taxid(g, s)
            parent = 100 + g
            if g == 6 and s < 10:
                parent = 30                               # species under a subgenus
            if g == 5 and s == 0:
                parent = 11                               # species straight under its family
            nodes.append((t, parent, "species"))
            tax.append(t)
    def seq(g, s):
        return sum(SPECIES[:g]) + s
    tax[seq(2, 1)] = species_taxid(2, 0)                  # taxids with two sequences
    tax[seq(3, 1)] = species_taxid(3, 0)
    for s, rank in ((1, "strain"), (2, "subspecies"), (3, "no rank")):
        leaf = 60000 + s
        nodes.append((leaf, species_taxid(5, s), rank))   # leaves under a species
        tax[seq(5, s)] = leaf
    nodes.append((60004, species_taxid(4, 4), "no rank"))
    tax[seq(4, 4)] = 60004
    nodes.append((60005, species_taxid(1, 0), "no rank"))   # a "no rank" leaf beside its species' own sequence
    tax[seq(1, 1)] = 60005
    tax[seq(5, 4)] = 105                                  # a sequence mapped to its genus
    tax[seq(5, 5)] = 77777                                # taxid missing from nodes.dmp
    tax[seq(5, 6)] = None                                 # sequence missing from the conversion table
    for i, _ in enumerate(COPIES):
        nodes.append((19000 + i, 190, "species"))
        tax.append(19000 + i)
    return tax, nodes, {species_taxid(5, 7), 21}


@functools.lru_cache(None)
def genomes():
    """(sequences as 0..3 arrays, {block name: (sequence ids holding it, its bases)}, repeat units)"""
    rng = np.random.default_rng(4242)
    fam_block = {f: rng.integers(0, 4, size=FAMILY_BLOCK, dtype=np.uint8) for f in (10,)}
    seqs, blocks = [], {}
    for g, S in enumerate(SPECIES):
        gb = rng.integers(0, 4, size=GENUS_BLOCK, dtype=np.uint8)
        ids = []
        for s in range(S):
            parts = [rng.integers(0, 4, size=500, dtype=np.uint8), gb, rng.integers(0, 4, size=500, dtype=np.uint8)]
            if FAMILY_OF[g] in fam_block:
                parts += [fam_block[FAMILY_OF[g]], rng.integers(0, 4, size=300, dtype=np.uint8)]
            ids.append(len(seqs))
            seqs.append(np.concatenate(parts))
        blocks["g%d" % g] = (tuple(ids), gb)
    blocks["f10"] = (tuple(i for g in range(4) for i in blocks["g%d" % g][0]), fam_block[10])
    units = []
    for c in COPIES:
        u = rng.integers(0, 4, size=REPEAT_UNIT, dtype=np.uint8)
        parts = []
        for _ in range(c):
            parts += [rng.integers(0, 4, size=REPEAT_GAP, dtype=np.uint8), u]
        parts.append(rng.integers(0, 4, size=REPEAT_GAP, dtype=np.uint8))
        units.append(u)
        seqs.append(np.concatenate(parts))
    return seqs, blocks, units


def write_fixture(d, build):
    """genomes.fa, conv.tsv, nodes.dmp, names.dmp of one build under d"""
    os.makedirs(d, exist_ok=True)
    seqs, _, _ = genomes()
    tax, nodes, unnamed = seq_taxonomy()
    pre = "cid" if build == "cid" else "seq"
    with open(os.path.join(d, "genomes.fa"), "wb") as f:
        for i, s in enumerate(seqs):
            f.write(b">%s%d\n" % (pre.encode(), i) + A[s].tobytes() + b"\n")
    with open(os.path.join(d, "conv.tsv"), "w") as f:
        for i, t in enumerate(tax):
            if t is not None:
                f.write("%s%d\t%d\n" % (pre, i, t))
    with open(os.path.join(d, "nodes.dmp"), "w") as f:
        for t, p, r in nodes:
            f.write("%d\t|\t%d\t|\t%s\t|\n" % (t, p, r))
    with open(os.path.join(d, "names.dmp"), "w") as f:
        for t, _, r in nodes:
            if t not in unnamed:
                f.write("%d\t|\t%s\t|\t\t|\tscientific name\t|\n" % (t, "root" if t == 1 else "%s %d" % (r.replace(" ", "_"), t)))
    return [os.path.join(d, x) for x in ("genomes.fa", "conv.tsv", "nodes.dmp", "names.dmp")]


@functools.lru_cache(None)
def index(build):
    """base name of the build's index: the committed golden copy (rewritten by the reference builder when recording)"""
    if util.RECORD:
        d = os.path.join(util.CACHE, "ties_record_" + build)
        fa, conv, nodes, names = write_fixture(d, build)
        base = os.path.join(d, "idx")
        util.build_cf([fa], conv, nodes, names, base, "ties_" + build)
        for k in "1234":
            with open("%s.%s.cf" % (base, k), "rb") as f, lzma.open(os.path.join(util.GOLDEN, "ties_%s.%s.cf.xz" % (build, k)), "wb", preset=9) as g:
                g.write(f.read())
    return util.golden_index("ties_" + build)


def project_build(build):
    """the same index written by the project's builder, which must write the recorded bytes (util.build_cf checks them)"""
    d = os.path.join(util.CACHE, "ties_project_" + build)
    fa, conv, nodes, names = write_fixture(d, build)
    base = os.path.join(d, "idx")
    util.build_cf([fa], conv, nodes, names, base, "ties_" + build)
    return base


# ----------------------------------------------------------------------------- reads
def revcomp(a):
    return np.frombuffer(a.tobytes()[::-1].translate(bytes.maketrans(b"ACGTN", b"TGCAN")), dtype=np.uint8)


def _piece(rng, src, lo, hi, sub=0.0):
    L = min(int(rng.integers(lo, hi + 1)), len(src))
    p = int(rng.integers(0, len(src) - L + 1))
    r = src[p:p + L].copy()
    if sub:
        m = rng.random(L) < sub
        r[m] = (r[m] + 1) & 3
    a = A[r].copy()
    return revcomp(a) if rng.random() < 0.5 else a


@functools.lru_cache(None)
def single_reads():
    """[(name, ascii bases)]: reads from every tie block, the family block and unique regions in the four length classes,
    random reads, reads across two tie groups and reads from each repeat unit"""
    seqs, blocks, units = genomes()
    rng = np.random.default_rng(77)
    out = []
    for b, (ids, bases) in blocks.items():
        for cls, (lo, hi) in LENGTHS.items():
            if lo > len(bases):
                continue
            for j in range(6):
                out.append(("%s_%s_%d" % (b, cls, j), _piece(rng, bases, lo, min(hi, len(bases)), 0.01 if j == 5 else 0.0)))
    for cls, (lo, hi) in LENGTHS.items():
        for j in range(16):
            si = int(rng.integers(0, len(seqs)))
            out.append(("u%d_%s_%d" % (si, cls, j), _piece(rng, seqs[si][:500], lo, min(hi, 500))))
            out.append(("rnd_%s_%d" % (cls, j), A[rng.integers(0, 4, size=int(rng.integers(lo, hi + 1)), dtype=np.uint8)].copy()))
    names = sorted(blocks)
    for j in range(24):
        x, y = names[j % len(names)], names[(j * 3 + 1) % len(names)]
        a, b = _piece(rng, blocks[x][1], 60, 200), _piece(rng, blocks[y][1], 60, 200)
        out.append(("span_%s_%s_%d" % (x, y, j), np.concatenate([a, b])))
    for i, u in enumerate(units):
        for j, L in enumerate((40, 64, 100, 100)):
            p = int(rng.integers(0, REPEAT_UNIT - L + 1))
            a = A[u[p:p + L]].copy()
            out.append(("rep%d_%d" % (COPIES[i], j), revcomp(a) if j % 2 else a))
    return out


@functools.lru_cache(None)
def pairs():
    """[(name, mate 1, mate 2)]: mates from two different tie groups, mate 2 the reverse complement of mate 1, and mates from
    a tie block with a unique-region partner"""
    seqs, blocks, _ = genomes()
    rng = np.random.default_rng(78)
    names = sorted(blocks)
    out = []
    for j in range(84):
        x, y = names[j % len(names)], names[(j * 5 + 2) % len(names)]
        lo, hi = list(LENGTHS.values())[j % 3]
        a = _piece(rng, blocks[x][1], lo, hi)
        if j % 3 == 0:
            b = revcomp(a)
        elif j % 3 == 1:
            b = _piece(rng, blocks[y][1], lo, hi)
        else:
            si = int(rng.integers(0, len(seqs)))
            b = _piece(rng, seqs[si][:500], lo, min(hi, 500))
        out.append(("p%d_%s_%s" % (j, x, y), a, b))
    return out


@functools.lru_cache(None)
def batches():
    se = single_reads()
    pr = pairs()
    return {"se": util.Batch([a for _, a in se]), "pe": util.Batch([a for _, a, _ in pr], [b for _, _, b in pr])}


OPTIONS = {
    "default": {}, "host": dict(host=HOST), "excl": dict(excl=EXCL), "genus": dict(rank_slot=2), "family": dict(rank_slot=3),
    "notraverse": dict(traverse=False), "minhit15": dict(min_hitlen=15),
}
CLI_OPTIONS = {"default": [], "host": ["--host-taxids", ",".join(map(str, HOST))], "genus": ["--classification-rank", "genus"]}
CLI_K = (2, 8, 16, 31, 32, 33, 64)
CLI_CASES = ("default", "host", "genus")


def mixed_reads():
    """(tie-free reads, reads that tie among 16, 31 and 32 sequences): the two parts of the "mixed" file, in that order"""
    se = single_reads()
    free = [r for r in se if r[0].startswith(("u", "rnd"))] * 16
    heavy = [r for r in se if r[0].startswith(("g2", "g3", "g4"))] * 12
    return free, heavy


def write_reads(d):
    """the read files: {input: centrifuge-class arguments}.  "mixed" has about 600 kB of tie-free reads and then about 250 kB of
    reads that tie among 16, 31 and 32 sequences: with 300 kB spans, the third span carries more tie sets than the first two
    predicted, so the host has to copy them again."""
    os.makedirs(d, exist_ok=True)
    se, pr = single_reads(), pairs()
    fq, fa = os.path.join(d, "se.fq"), os.path.join(d, "se.fa")
    p1, p2 = os.path.join(d, "pe_1.fq"), os.path.join(d, "pe_2.fq")
    util.synth.write_fastq(fq, se)
    util.synth.write_fasta(fa, se)
    util.synth.write_fastq(p1, [(n, a) for n, a, _ in pr])
    util.synth.write_fastq(p2, [(n, b) for n, _, b in pr], qual=b"5")
    free, heavy = mixed_reads()
    mixed = os.path.join(d, "mixed.fa")
    util.synth.write_fasta(mixed, [("m%d_%s" % (i, n), a) for i, (n, a) in enumerate(free + heavy)])
    return {"se_fq": ["-q", "-U", fq], "se_fa": ["-f", "-U", fa], "pe_fq": ["-q", "-1", p1, "-2", p2], "mixed": ["-f", "-U", mixed]}


def cli_key(build, inp, k, case):
    return "ties/%s/%s/k%d/%s" % (build, inp, k, case)
