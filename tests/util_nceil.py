"""Inputs and recorded reference outputs of the --n-ceil tests.  The digests follow util.reference's scheme (SHA-256 of
what the unmodified reference wrote, re-recorded with CFB_RECORD_REFERENCE=1) in a file of their own,
tests/golden/n_ceil_digests.json.  Also a restatement of the reference's ceiling (SimpleFunc::f<size_t>, simple_func.h)
in plain Python floats, independent of centrifuge_b200/csrc/cf_nceil.h."""
import atexit
import gzip
import json
import math
import os
import random
import subprocess
import sys

import numpy as np

import util

DIGESTS = os.path.join(util.GOLDEN, "n_ceil_digests.json")
_digests = None
_recorded = {}

# --n-ceil values of the tests (None: the option is not given); C,1e30 is past 2^64, where the reference's size_t
# conversion gives 0
CEILS = [None, "C,0", "0", "L,0,0", "L,0,1", "C,1e9", "L,2,0.05", "S,1,2", "G,0,3", "C,-3", "L,abc", "C,1e30", "S,1", "G,2", "L,1"]
BAD_CEILS = ["X,1", "1,2,3,4", ",5"]
# an empty value is not refused: tokenize keeps one empty token, so it reads as "C," -- a constant ceiling of 0
QUIRK_FLAGS = [["--ignore-quals"], ["--nofw"], ["--norc"], ["--ignore-quals", "--nofw", "--norc"]]


def reference(key, run):
    global _digests
    key = "n_ceil/" + key
    if util.RECORD:
        if not util.have_ref():
            raise RuntimeError("CFB_RECORD_REFERENCE=1 needs the reference binaries under oracle/_ref (make -C oracle ref)")
        d = util.digest(run())
        if not _recorded:
            atexit.register(_save)
        _recorded[key] = d
        return d
    if _digests is None:
        with open(DIGESTS) as f:
            _digests = json.load(f)
    if key not in _digests:
        raise KeyError("no recorded reference output for %r (re-record, see tests/util.py)" % key)
    return _digests[key]


def _save():
    old = {}
    if os.path.exists(DIGESTS):
        with open(DIGESTS) as f:
            old = json.load(f)
    old.update(_recorded)
    with open(DIGESTS, "w") as f:
        json.dump(old, f, indent=0, sort_keys=True)
        f.write("\n")


# ----------------------------------------------------------------------------- the reference's ceiling, restated
# (type, constant, coefficient) each CEILS entry parses to in the reference: PARSE_FUNC (aligner_seed_policy.cpp:47-75)
# on top of SimpleFunc::init(L, 0, DBL_MAX, 0, 0.15f) (aligner_seed_policy.cpp:296-298), so a coefficient left unset is
# the float 0.15f widened (F15), and `istringstream >> double` gives 0 for "abc".  Without the option the product keeps
# the double 0.15, which gives the reference's 0.15f ceiling for every length below 8 388 613 bases.
F15 = float(np.float32(0.15))
PARSED = {None: (2, 0.0, 0.15), "C,0": (1, 0.0, F15), "0": (1, 0.0, F15), "L,0,0": (2, 0.0, 0.0), "L,0,1": (2, 0.0, 1.0),
          "C,1e9": (1, 1e9, F15), "L,2,0.05": (2, 2.0, 0.05), "S,1,2": (3, 1.0, 2.0), "G,0,3": (4, 0.0, 3.0),
          "C,-3": (1, -3.0, F15), "L,abc": (2, 0.0, F15), "C,1e30": (1, 1e30, F15), "": (1, 0.0, F15),
          "S,1": (3, 1.0, F15), "G,2": (4, 2.0, F15), "L,1": (2, 1.0, F15)}


def ceiling(f, n):
    """SimpleFunc::f<size_t>((double)n) with min 0 and max DBL_MAX, x86-64 size_t conversion."""
    t, c, l = f
    x = float(n)
    g = 0.0 if t == 1 else (x if t == 2 else (math.sqrt(x) if t == 3 else (math.log(x) if x > 0 else -math.inf)))
    with_nan = l * g
    v = c + with_nan
    lo = v if v < sys.float_info.max else sys.float_info.max
    r = lo if 0.0 < lo else 0.0
    if r == sys.float_info.max:
        return 2 ** 64 - 1
    if r >= 2.0 ** 64:
        return 0
    return int(r)


def passes(f, seq):
    """nFilter + lenfilt of a mate given as ASCII (N and '.' count)"""
    if len(seq) < 2:
        return False
    ns = sum(1 for ch in seq if ch in "Nn.")
    return ns <= ceiling(f, len(seq))


# ----------------------------------------------------------------------------- inputs
def _ndense(rng, s, mode):
    s = list(s)
    n = len(s)
    if mode == 1:                                  # N runs at both ends
        k = rng.randint(1, max(1, n // 4))
        for i in range(min(k, n)):
            s[i] = "N"
            s[n - 1 - i] = "N"
    elif mode == 2:                                # one N every 10-mer window
        for i in range(rng.randint(0, 9), n, 10):
            s[i] = "N"
    elif mode == 3:                                # every 2nd base
        for i in range(0, n, 2):
            s[i] = "N"
    elif mode == 4:                                # every 3rd base, as '.'
        for i in range(0, n, 3):
            s[i] = "."
    elif mode == 5:                                # all N
        s = ["N"] * n
    elif mode == 6:                                # a handful
        for _ in range(rng.randint(1, 6)):
            s[rng.randrange(n)] = "N"
    return "".join(s)


def make_reads(seed=7):
    """(single reads, mate-1 reads, mate-2 reads): lists of (name, ASCII sequence) drawn from the adv index's reads"""
    rng = random.Random(seed)
    src = [a.tobytes().decode() for n, a in util.parse_reads(_adv_reads()) if len(a) >= 40]
    genome = "".join(src)
    singles = []
    for i in range(360):
        s = src[i % len(src)]
        singles.append(("s%d" % i, _ndense(rng, s, i % 7)))
    for L in (1, 2, 10, 100, 321):
        for mode in (0, 1, 2, 3, 5):
            s = (genome[rng.randrange(len(genome) - 400):][:L])
            singles.append(("len%d_%d" % (L, mode), _ndense(rng, s, mode)))
    for L in (60000, 60001):
        for mode in (0, 3):
            o = rng.randrange(len(genome) - L) if len(genome) > L else 0
            s = (genome * (L // len(genome) + 2))[o:o + L]
            singles.append(("long%d_%d" % (L, mode), _ndense(rng, s, mode)))
    m1, m2 = [], []
    for i in range(240):
        a, b = src[(2 * i) % len(src)], src[(2 * i + 1) % len(src)]
        ma, mb = (i % 7, 0) if i % 2 else (0, i % 7)    # one mate N-dense, the other clean
        m1.append(("p%d/1" % i, _ndense(rng, a, ma)))
        m2.append(("p%d/2" % i, _ndense(rng, b, mb)))
    return singles, m1, m2


def _adv_reads():
    import lzma
    fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
    if not os.path.exists(fa):
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa + ".tmp", "wb") as g:
            g.write(f.read())
        os.replace(fa + ".tmp", fa)
    return fa


def fastq(reads):
    return "".join("@%s\n%s\n+\n%s\n" % (n, s, "".join(chr(33 + (i * 7 + len(n)) % 40) for i in range(len(s)))) for n, s in reads).encode()


def fasta(reads):
    return "".join(">%s\n%s\n" % (n, s) for n, s in reads).encode()


def write_inputs(d):
    """The input sets under d: name -> CLI read arguments.  'se' is strict FASTQ (the text operator takes it whole)."""
    singles, m1, m2 = make_reads()
    os.makedirs(d, exist_ok=True)
    files = {"se.fq": fastq(singles), "se.fa": fasta(singles), "p1.fq": fastq(m1), "p2.fq": fastq(m2),
             "empty.fq": fastq([(n, s) for n, s in singles[:40]] + [("e0", "ACGTNACGTACGTAAGT"), ("e1", ""), ("e2", "NNNNNNNNNN"),
                                ("e3", "A"), ("e4", "N"), ("e5", "NA"), ("e6", "")] + [(n, s) for n, s in singles[40:80]])}
    for k, v in files.items():
        p = os.path.join(d, k)
        if not os.path.exists(p):
            with open(p, "wb") as f:
                f.write(v)
    for name in ("se.fq", "se.fa"):
        gz = os.path.join(d, name + ".gz")
        if not os.path.exists(gz):
            with open(gz, "wb") as f:
                f.write(gzip.compress(files[name], 6, mtime=0))
    j = lambda k: os.path.join(d, k)  # noqa: E731
    return {"se": ["-U", j("se.fq")], "fa": ["-f", "-U", j("se.fa")], "gz": ["-U", j("se.fq.gz")], "fagz": ["-f", "-U", j("se.fa.gz")],
            "pe": ["-1", j("p1.fq"), "-2", j("p2.fq")], "empty": ["-U", j("empty.fq")]}


def ceil_args(spec):
    return [] if spec is None else ["--n-ceil", spec]


def ceil_key(spec):
    return "default" if spec is None else "c[" + spec + "]"


def run_cli(binary, args, tmp, env=None):
    """(TSV bytes, report bytes) of a run"""
    return util.run_cli(binary, args, os.path.join(str(tmp), "o.tsv"), os.path.join(str(tmp), "o.rep"), env=env)


def error_of(binary, spec):
    """(exit code, first stderr line) of a run refused for its --n-ceil value"""
    p = subprocess.run([binary, "--n-ceil", spec, "-x", "/nonexistent/idx", "-U", "/nonexistent/r.fq"],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    return p.returncode, p.stderr.decode().split("\n", 1)[0]


def ref_kreport(base, args, tmp):
    """The reference's Kraken-style report of a run: its Perl centrifuge-kreport over the binary's TSV (recording only)"""
    run_cli(util.REF_CLASS, ["-x", base] + args, tmp)
    p = subprocess.run(["perl", util.ref_script("centrifuge-kreport", tmp), "-x", base, os.path.join(str(tmp), "o.tsv")],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True)
    return p.stdout


# the reference inputs of each input set ("gz" / "fagz" hold the bytes of "se" / "fa"; the binary is built without zlib)
REF_OF = {"gz": "se", "fagz": "fa"}
