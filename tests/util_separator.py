"""Inputs and recorded reference outputs of the --separator tests.  The digests follow util.reference's scheme (SHA-256 of
what the unmodified reference wrote, re-recorded with CFB_RECORD_REFERENCE=1) in a file of their own,
tests/golden/separator_digests.json."""
import atexit
import glob
import json
import os
import re
import subprocess

import util

DIGESTS = os.path.join(util.GOLDEN, "separator_digests.json")
SEP = b"#File_End_Here\n"
_digests = None
_recorded = {}


def reference(key, run):
    """Digest of what the reference produced for the case named `key`; run() produces that output with the reference
    and is called only when recording."""
    global _digests
    key = "separator/" + key
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


# ----------------------------------------------------------------------------- inputs
def fastq(reads, crlf=False):
    nl = b"\r\n" if crlf else b"\n"
    return b"".join(b"@" + n.encode() + nl + a.tobytes() + nl + b"+" + nl + b"I" * len(a) + nl for n, a in reads)


def adv_regular_reads(adv_reads):
    return [(n, a) for n, a in util.parse_reads(adv_reads) if len(a) > 0 and n]


# Two -1/-2 pairs, then three -U files: the second -U file is empty and the first has CR-LF line ends.  All reads are
# drawn from the same genera of the adv index, so tie sets of earlier inputs weigh in later inputs' abundances.
INPUTS = [("p0", (0, 300), (300, 600)), ("p1", (600, 800), (800, 1000)), ("u0", (1000, 1400), None), ("u1", None, None),
          ("u2", (1400, 2000), None)]
CRLF = {"u0"}


def write_inputs(d, reads, ext=""):
    """INPUTS as FASTQ files under d: ([(mate-1 or single file, mate-2 file or None)] in processing order, CLI args).
    ext ".gz" / ".bz2" compresses every file."""
    import bz2
    import gzip
    files, args, m1, m2, singles = [], [], [], [], []
    for tag, a, b in INPUTS:
        paths = []
        for k, rng in enumerate((a, b) if b else (a,)):
            data = fastq(reads[rng[0]:rng[1]] if rng else [], crlf=tag in CRLF)
            if ext == ".gz":
                data = gzip.compress(data, 6)
            elif ext == ".bz2":
                data = bz2.compress(data, 9)
            p = os.path.join(str(d), "%s_%d.fq%s" % (tag, k + 1, ext) if b else "%s.fq%s" % (tag, ext))
            with open(p, "wb") as f:
                f.write(data)
            paths.append(p)
        files.append((paths[0], paths[1] if b else None))
        if b:
            m1.append(paths[0]); m2.append(paths[1])
        else:
            singles.append(paths[0])
    args = ["-1", ",".join(m1), "-2", ",".join(m2), "-U", ",".join(singles)]
    return files, args


# ----------------------------------------------------------------------------- runs
def stderr_lines(err):
    """The stderr lines a --separator run's digest covers: each report's name and the EM's two lines."""
    return [ln for ln in err.decode().splitlines() if ln.startswith("report file ") or "EM algorithm" in ln or "Probability diff" in ln]


def reports(cwd):
    """[(name, bytes)] of the per-input reports in cwd, by input index"""
    names = sorted((int(re.match(r".*centrifuge_report_(\d+)\.tsv$", p).group(1)), p) for p in glob.glob(os.path.join(str(cwd), "centrifuge_report_*.tsv")))
    return [(os.path.basename(p), open(p, "rb").read()) for _, p in names]


def run(exe, args, cwd, out="out.tsv", env=None):
    """exe --separator args, run in the fresh directory cwd with -S out (or "-": stdout) and --report-file rep.tsv:
    ((TSV, reports, stderr lines), whether rep.tsv was written, the whole stderr)."""
    os.makedirs(str(cwd), exist_ok=True)
    p = subprocess.run([exe, "--separator"] + list(args) + ["-S", out, "--report-file", "rep.tsv"], cwd=str(cwd),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    assert p.returncode == 0, p.stderr.decode()[-3000:]
    tsv = p.stdout if out == "-" else open(os.path.join(str(cwd), out), "rb").read()
    return (tsv, reports(cwd), stderr_lines(p.stderr)), os.path.exists(os.path.join(str(cwd), "rep.tsv")), p.stderr.decode()


def reference_outputs(key, args, tmp):
    """Recorded digests of the reference's --separator run with args: (digest of (TSV, reports, stderr lines), digest of
    whether the --report-file was written)."""
    got = {}

    def ref():
        if "r" not in got:
            got["r"] = run(util.REF_CLASS, args, os.path.join(str(tmp), "ref_" + key.replace("/", "_")))
        return got["r"]
    return reference(key, lambda: ref()[0]), reference(key + "/report_file_written", lambda: ref()[1])
