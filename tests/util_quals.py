"""Inputs and recorded reference outputs of the quality-encoding tests (--phred64, --solexa-quals, --int-quals and their
aliases).  The digests follow util.reference's scheme (SHA-256 of what the unmodified reference wrote, re-recorded with
CFB_RECORD_REFERENCE=1) in a file of their own, tests/golden/quals_digests.json.  Also a restatement of the reference's
conversions (charToPhred33 / intToPhred33, qual.h:105-171, and the published Solexa -> Phred formula) in plain Python,
independent of centrifuge_b200/csrc/cf_quals.h."""
import atexit
import gzip
import json
import math
import os
import random
import subprocess

import util

DIGESTS = os.path.join(util.GOLDEN, "quals_digests.json")
_digests = None
_recorded = {}


def reference(key, run):
    global _digests
    key = "quals/" + key
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


# ----------------------------------------------------------------------------- the reference's conversions, restated
def solexa_to_phred(q):
    """round(10 log10(1 + 10^(q/10))), 0 below -10; 255 past 255 (where the reference reads past its table)"""
    if q < -10:
        return 0
    q = min(q, 255)
    return int(math.floor(10.0 * math.log10(1.0 + 10.0 ** (q / 10.0)) + 0.5))


def signed(b):
    return b - 256 if b >= 128 else b


def char_to_phred33(b, solexa, phred64):
    """phred33 value of a kept quality byte, or None where the reference refuses it (a space is refused before)"""
    c = signed(b)
    if solexa:
        return solexa_to_phred(c - 64) + 33
    if phred64:
        return None if c < 64 else c - 31
    return None if c < 33 else c


def int_to_phred33(v, solexa):
    """intToPhred33 before its char conversion: below 33 is the "Saw negative Phred quality" refusal"""
    return solexa_to_phred(v) + 33 if solexa else min(v, 93) + 33


# ----------------------------------------------------------------------------- modes
# name -> (options in command-line order, how the quality lines of its inputs are written)
MODES = {
    "phred64": (["--phred64"], "p64"),
    "phred64-quals": (["--phred64-quals"], "p64"),
    "solexa1.3-quals": (["--solexa1.3-quals"], "p64"),
    "solexa-quals": (["--solexa-quals"], "sol"),
    "int-quals": (["--int-quals"], "int"),
    "integer-quals": (["--integer-quals"], "int"),
    "phred33": (["--phred33"], "p33"),
    "phred33-quals": (["--phred33-quals"], "p33"),
    "phred64+phred33": (["--phred64", "--phred33"], "p33"),
    "solexa-quals+phred64": (["--solexa-quals", "--phred64"], "sol"),
    "int-quals+solexa-quals": (["--int-quals", "--solexa-quals"], "intsol"),
    "int-quals+phred64": (["--int-quals", "--phred64"], "int"),
}
# one mode per way of writing the qualities: the input sets are run under these
MAIN = ["phred64", "solexa-quals", "int-quals", "int-quals+solexa-quals", "phred33"]


def opt_names(mode):
    """the mode's options without dashes, comma-separated, as cfb_test_parse_quals takes them"""
    return ",".join(o.lstrip("-") for o in MODES[mode][0])


def is_int(mode):
    return MODES[mode][1] in ("int", "intsol")


# value range of each way of writing, and how a value is written
_RANGE = {"p33": (0, 60), "p64": (0, 62), "sol": (-31, 62), "int": (0, 60), "intsol": (-15, 60)}


def render(kind, vals):
    if kind == "p33":
        return bytes(33 + v for v in vals)
    if kind in ("p64", "sol"):
        return bytes(64 + v for v in vals)
    return " ".join(str(v) for v in vals).encode()


def _vals(rng, kind, n):
    lo, hi = _RANGE[kind]
    return [rng.randint(lo, hi) for _ in range(n)]


def _adv_reads():
    import lzma
    fa = os.path.join(util.CACHE, "golden", "adv.reads.fa")
    if not os.path.exists(fa):
        os.makedirs(os.path.dirname(fa), exist_ok=True)
        with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(fa + ".tmp", "wb") as g:
            g.write(f.read())
        os.replace(fa + ".tmp", fa)
    return [a.tobytes() for _, a in util.parse_reads(fa) if len(a) >= 40]


def _name(i, prefix="r"):
    return ("%s%d" % (prefix, i) + (" desc x" if i % 7 == 3 else "") + ("/1" if i % 5 == 2 else "")).encode()


def fastq(recs):
    return b"".join(b"@" + n + b"\n" + s + b"\n+\n" + q + b"\n" for n, s, q in recs)


def records(kind, which, seed=11):
    """[(name, bases, quality line)] of an input set written in `kind`"""
    rng = random.Random(seed * 1000 + sum(map(ord, kind + which)))
    src = _adv_reads()
    if which in ("se", "trim"):
        out = []
        for i in range(400):
            s = src[i % len(src)]
            v = _vals(rng, kind, len(s) + (1 if i % 9 == 4 else 0))            # some one longer than the read
            q = render(kind, v)
            if which == "trim" and i % 4 == 1 and kind in ("p33", "p64"):     # a refused character inside the 5' trim
                q = b"\x1f" + q[1:] if kind == "p33" else b"5" + q[1:]
            out.append((_name(i), s, q))
        return out
    if which in ("p1", "p2"):
        off = 0 if which == "p1" else 1
        return [(("p%d/%d" % (i, off + 1)).encode(), src[(2 * i + off) % len(src)],
                 render(kind, _vals(rng, kind, len(src[(2 * i + off) % len(src)])))) for i in range(200)]
    if which == "quirks":                                                      # integer lines only
        out = []
        top = [93, 94, 100, 150] if kind == "int" else [93, 94, 100, 230, 255]
        for i in range(120):
            s = src[i % len(src)]
            v = _vals(rng, kind, len(s) + (1 if i % 3 == 0 else 0))
            toks = [str(x) for x in v]
            k = i % 8
            if k == 1:
                toks[2] = "\t" + toks[2]                         # atoi skips a tab
            elif k == 2:
                toks[3] = "+" + toks[3]                          # a sign
            elif k == 3:
                toks[4] = toks[4] + "x9"                         # stops at the first non-digit
            elif k == 4:
                toks[5] = str(top[i % len(top)])                 # 93 and above
                toks[6] = str(top[(i + 1) % len(top)])
            elif k == 5:
                toks[1] = "000" + toks[1]
            line = " ".join(toks)
            if k == 6:
                line = " " + " ".join(toks[:-1])                 # a leading space: an empty first token (0)
            elif k == 7:
                line = line.replace(" ", "   ", 5) + "  "         # runs of spaces and trailing ones give no tokens
            out.append((_name(i), s, line.encode()))
        return out
    if which == "long":
        out = [(_name(i), src[i], render(kind, _vals(rng, kind, len(src[i])))) for i in range(30)]
        if kind in ("int", "intsol"):
            # integer lines of 4095 bytes and more: gets takes 4095 bytes, drops the next one and leaves the rest of the
            # line in the stream -- here a 4200-byte line, whose last 104 bytes become the next record's name
            s = (src[0] * 20)[:1000]
            out.append((b"long1", s, (" ".join(["30"] * 1000) + " " * 1201).encode()))
        else:
            s = (b"".join(src) * 4)[:60001]                                                # a long unit
            out.append((b"long60001", s, render(kind, _vals(rng, kind, len(s)))))
        out += [(_name(i, "t"), src[i + 30], render(kind, _vals(rng, kind, len(src[i + 30])))) for i in range(30)]
        return out
    if which == "line4096":                                                    # integer lines of 4094, 4095 and 4096 bytes
        out = [(_name(i), src[i], render(kind, _vals(rng, kind, len(src[i])))) for i in range(20)]
        for k, pad in enumerate((1095, 1096, 1097)):
            s = (src[k] * 20)[:1000]
            out.append((("line%d" % (2999 + pad)).encode(), s, (" ".join(["30"] * 1000) + " " * pad).encode()))
            out += [(_name(i, "u%d_" % k), src[i], render(kind, _vals(rng, kind, len(src[i])))) for i in range(20, 30)]
        return out
    raise KeyError(which)


# each refusal: (mode, trims, what the one bad record's quality line is)
ERRORS = {
    "phred64_below_64": ("phred64", (0, 0)),
    "phred64_space": ("phred64", (0, 0)),
    "solexa_space": ("solexa-quals", (0, 0)),
    "int_negative": ("int-quals", (0, 0)),
    "int_negative_in_5p_trim": ("int-quals", (3, 0)),
    "int_too_few": ("int-quals", (0, 0)),
    "int_too_many": ("int-quals", (0, 0)),
    "intsol_too_many": ("int-quals+solexa-quals", (0, 0)),
}


def error_records(case):
    mode, _ = ERRORS[case]
    kind = MODES[mode][1]
    rng = random.Random(5)
    src = _adv_reads()
    out = [(_name(i), src[i], render(kind, _vals(rng, kind, len(src[i])))) for i in range(60)]
    s = src[61]
    v = _vals(rng, kind, len(s))
    q = render(kind, v)
    if case == "phred64_below_64":
        q = q[:10] + b"5" + q[11:]
    elif case.endswith("_space"):
        q = q[:10] + b" " + q[11:]
    elif case == "int_negative":
        q = render(kind, v[:7] + [-3] + v[8:])
    elif case == "int_negative_in_5p_trim":
        q = render(kind, [-2] + v[1:])
    elif case == "int_too_few":
        q = render(kind, v[:-1])
    elif case in ("int_too_many", "intsol_too_many"):
        q = render(kind, v + [20, 20])
    out.append((b"bad", s, q))
    out += [(_name(i, "z"), src[i], render(kind, _vals(rng, kind, len(src[i])))) for i in range(60, 100)]
    return out


def write(path, data):
    if not os.path.exists(path):
        with open(path + ".tmp", "wb") as f:
            f.write(data)
        os.replace(path + ".tmp", path)
    return path


def inputs(d, mode):
    """The input sets of a mode under d: name -> CLI read arguments"""
    kind = MODES[mode][1]
    os.makedirs(d, exist_ok=True)
    j = lambda k: os.path.join(d, "%s.%s" % (kind, k))  # noqa: E731
    se = fastq(records(kind, "se"))
    out = {"se": ["-U", write(j("se.fq"), se)],
           "gz": ["-U", write(j("se.fq.gz"), gzip.compress(se, 6, mtime=0))],
           "pe": ["-1", write(j("p1.fq"), fastq(records(kind, "p1"))), "-2", write(j("p2.fq"), fastq(records(kind, "p2")))],
           "trim": ["-5", "3", "-3", "2", "-U", write(j("trim.fq"), fastq(records(kind, "trim")))],
           "long": ["-U", write(j("long.fq"), fastq(records(kind, "long")))],
           "fa": ["-f", "-U", write(os.path.join(d, "se.fa"), b"".join(b">" + n + b"\n" + s + b"\n" for n, s, _ in records("p33", "se")))]}
    if kind in ("int", "intsol"):
        out["quirks"] = ["-U", write(j("quirks.fq"), fastq(records(kind, "quirks")))]
        out["line4096"] = ["-U", write(j("line4096.fq"), fastq(records(kind, "line4096")))]
    return out


# the reference inputs of each set ("gz" holds the bytes of "se"; the binary is built without zlib)
REF_OF = {"gz": "se"}
QCOLS = "readID,readSeq,readQual,QUAL,readQual2"


def error_lines(stderr):
    """the refusal's lines: the reference's reader messages start with Error, Saw or Try"""
    return [l for l in stderr.decode(errors="replace").splitlines() if l.startswith(("Error", "Saw", "Try"))]


def run_ref_error(binary, base, args, tmp):
    """(failed, error lines, TSV or b"") of a run that may be refused"""
    tsv = os.path.join(str(tmp), "e.tsv")
    p = subprocess.run([binary, "-x", base] + args + ["-S", tsv, "--report-file", os.path.join(str(tmp), "e.rep")],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    failed = p.returncode != 0
    out = b""
    if not failed:
        with open(tsv, "rb") as f:
            out = f.read()
    return failed, error_lines(p.stderr), out
