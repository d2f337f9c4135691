"""--tab-fmt-cols and --passthrough on the CPU: option parsing against the unmodified reference binary, and the host
formatter (cfb_test_host_path_cols) on random column lists around oracle records, byte for byte against the reference's
TSV for the same files and options (by their recorded digest).  Also holds a restatement of the `centrifuge` wrapper's
read split (--un / --al / --un-conc / --al-conc / --no-unal), checked against the real wrapper where the reference tree
is present."""
import ctypes as C
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import util
import util_cols
from test_classify_fuzz import API_OPTS, CLI_OPTS, make_reads
from util_fuzz import clean_reads

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
NAMES = ["readID", "seqID", "taxID", "taxRank", "taxLevel", "taxName", "score", "2ndBestScore", "hitLength", "queryLength",
         "numMatches", "readSeq", "readQual", "readSeq1", "SEQ1", "readSeq2", "SEQ2", "readQual1", "QUAL1", "readQual2", "QUAL2",
         "QNAME", "FLAG", "RNAME", "POS", "MAPQ", "CIGAR", "RNEXT", "PNEXT", "TLEN", "SEQ", "QUAL"]
DEFAULT = "readID,seqID,taxID,score,2ndBestScore,hitLength,queryLength,numMatches"
WRAPPER = DEFAULT + ",readSeq,readQual"


# ----------------------------------------------------------------------------- the wrapper's split, restated
def perl_split(s, sep):
    """Perl's split on a literal separator: trailing empty fields are dropped."""
    v = s.split(sep)
    while v and v[-1] == b"":
        v.pop()
    return v


def wrapper_split(stdout, fns, no_unal=False):
    """What the `centrifuge` script (centrifuge:778-934) writes from centrifuge-class's stdout: {name: bytes} for the TSV
    ("out") and the read files of `fns` (a set of "un", "al", "un-conc", "al-conc"; the conc ones as "<name>1" and
    "<name>2").  With read files the wrapper has asked for `--tab-fmt-cols <default>,readSeq,readQual --passthrough` and
    strips the last two columns again; with --no-unal alone it has added only --passthrough."""
    lines = stdout.split(b"\n")
    header, rows = lines[0], lines[1:]
    if rows and rows[-1] == b"":
        rows = rows[:-1]
    cols = header.split(b"\t")
    strip = bool(fns)
    seq_i = qual_i = id_i = -1
    for i, c in enumerate(cols):
        if b"readSeq" in c:
            seq_i = i
        elif b"readQual" in c:
            qual_i = i
        elif b"readID" in c:
            id_i = i
    out = {"out": [(b"\t".join(perl_split(header, b"\t")[:-2]) if strip else header) + b"\n"]}
    for k in fns:
        if k.endswith("conc"):
            out[k + "1"], out[k + "2"] = [], []
        else:
            out[k] = []
    for row in rows:
        c = perl_split(row, b"\t")
        unal = b"unclassified" in row
        if row[:1] != b"#" and fns and seq_i >= 0:
            pair = b"_" in c[seq_i]
            if not pair and ("un" in fns or "al" in fns):
                f = lambda i: c[i] if i < len(c) else b""
                rec = (b"@" + f(id_i) + b"\n" + f(seq_i) + b"\n+\n" + f(qual_i) + b"\n") if qual_i >= 0 else (b">" + f(id_i) + b"\n" + f(seq_i) + b"\n")
                k = "un" if unal else "al"
                if k in fns:
                    out[k].append(rec)
            if pair and ("un-conc" in fns or "al-conc" in fns):
                s = perl_split(c[seq_i], b"_")
                s1, s2 = (s[0] if s else b""), (s[1] if len(s) > 1 else b"")
                q = c[qual_i] if qual_i < len(c) else b""
                q1, q2 = q[:len(s1)], q[len(s1) + 1:]
                k = "un-conc" if unal else "al-conc"
                if k in fns:
                    out[k + "1"].append(b"@" + c[id_i] + b"\n" + s1 + b"\n+\n" + q1 + b"\n")
                    out[k + "2"].append(b"@" + c[id_i] + b"\n" + s2 + b"\n+\n" + q2 + b"\n")
        if not (no_unal and unal):
            out["out"].append((b"\t".join(c[:-2]) if strip else row) + b"\n")
    return {k: b"".join(v) for k, v in out.items()}


WRAPPER_MODES = {"un": ["--un", "{d}/un.fq"], "al": ["--al", "{d}/al.fq"], "un-conc": ["--un-conc", "{d}/uc.fq"],
                 "al-conc": ["--al-conc", "{d}/ac.fq"], "no-unal": ["--no-unal"]}


def wrapper_files(mode, d):
    """Files the wrapper writes for one mode, in the order wrapper_split names them."""
    return {"un": {"un": d + "/un.fq"}, "al": {"al": d + "/al.fq"}, "un-conc": {"un-conc1": d + "/uc.1.fq", "un-conc2": d + "/uc.2.fq"},
            "al-conc": {"al-conc1": d + "/ac.1.fq", "al-conc2": d + "/ac.2.fq"}, "no-unal": {}}[mode]


def run_real_wrapper(tmp, args, mode):
    """Recording only: the reference's Perl `centrifuge` beside the reference centrifuge-class (copied, since the script
    resolves its own directory), run with `mode`; returns {name: bytes} for stdout ("out") and every file it wrote."""
    stage = os.path.join(str(tmp), "wrap")
    os.makedirs(stage, exist_ok=True)
    src = os.path.join(util.REF_TREE, "centrifuge")
    if not os.path.exists(src):
        raise RuntimeError("recording needs the reference's sources (no %s; set CFB_REFERENCE_TREE)" % src)
    shutil.copy(src, os.path.join(stage, "centrifuge"))
    shutil.copy(util.REF_CLASS, os.path.join(stage, "centrifuge-class"))
    od = os.path.join(str(tmp), "wout_" + mode)
    os.makedirs(od, exist_ok=True)
    extra = [a.format(d=od) for a in WRAPPER_MODES[mode]]
    p = subprocess.run(["perl", os.path.join(stage, "centrifuge")] + args + extra + ["--report-file", os.path.join(od, "rep")],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, check=True)
    out = {"out": p.stdout}
    for k, f in wrapper_files(mode, od).items():
        out[k] = open(f, "rb").read()
    return out


def wrapper_cols(mode):
    """The column option the wrapper adds to centrifuge-class's command line for one mode (besides --passthrough)."""
    return [] if mode == "no-unal" else ["--tab-fmt-cols", WRAPPER]


def split_for(mode, stdout):
    """wrapper_split for one mode, keyed as run_real_wrapper keys its files."""
    fns = set() if mode == "no-unal" else {mode}
    got = wrapper_split(stdout, fns, no_unal=mode == "no-unal")
    return {k: got[k] for k in ["out"] + sorted(wrapper_files(mode, "."))}


# ----------------------------------------------------------------------------- option parsing
PARSE_CASES = [",".join(NAMES), "readID", "readID,,taxID", "readID,taxID,", ",readID", "", ",", "readID,bogus,taxID", "readid",
               "readID, taxID", "SEQ1,SEQ2,QUAL1,QUAL2,CIGAR,FLAG"]


def _reads_fa(tmp):
    p = str(tmp / "one.fa")
    with open(p, "wb") as f:
        f.write(b">r1\nACGTACGTACGTACGTACGTACGTACGTAC\n")
    return p


@pytest.mark.parametrize("i", range(len(PARSE_CASES)))
def test_column_list_parsing_matches_reference(i, tmp_path):
    """Exit code, message and header line of the reference for one --tab-fmt-cols value (and, for the last cases, the
    option given twice: the last one wins, an invalid one anywhere stops the run)."""
    util.ensure_oracle()
    base = util.golden_index("adv")
    fa = _reads_fa(tmp_path)
    cols = PARSE_CASES[i]
    lists = [cols] if i < 7 else [("readID" if i % 2 else "bogus2"), cols]     # given twice: the last one wins, a bad one stops the run

    def run(exe, extra):
        args = sum((["--tab-fmt-cols", c] for c in lists), [])
        p = subprocess.run([exe, "-f", "-x", base, "-U", fa, "-S", str(tmp_path / "o.tsv"), "--report-file", str(tmp_path / "o.rep")] + args + extra,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        errs = [l for l in p.stderr.decode().splitlines() if l.startswith("Column definition")]
        return p.returncode, errs
    rc, errs = run(EXE, ["--arg-desc"])      # option parsing only: --arg-desc ends the run once every option before it is read
    header = None
    if rc == 0:
        lib = C.CDLL(util.PRODUCT_LIB)
        out = str(tmp_path / "h.tsv")
        rec_off = np.zeros(2, dtype=np.uint32)
        assert lib.cfb_test_host_path_cols(base.encode(), fa.encode(), None, 1, 5, C.c_uint32(0), 0, 0, rec_off.ctypes.data_as(C.POINTER(C.c_uint32)),
                                           None, C.c_uint64(1), lists[-1].encode(), out.encode(), str(tmp_path / "h.rep").encode(), None) == 0
        header = open(out, "rb").read().split(b"\n")[0]

    def ref():
        rrc, rerrs = run(util.REF_CLASS, [])
        return rrc, rerrs, (open(str(tmp_path / "o.tsv"), "rb").read().split(b"\n")[0] if rrc == 0 else None)
    util.assert_matches((rc, errs, header), util_cols.reference("tab_cols/parse/%d" % i, ref), lists)


def test_arg_desc_lists_the_new_options():
    p = subprocess.run([EXE, "--arg-desc"], stdout=subprocess.PIPE, check=True)
    lines = p.stdout.decode().splitlines()
    assert "tab-fmt-cols\t1" in lines and "passthrough\t0" in lines


def test_kreport_needs_its_columns(tmp_path):
    base = util.golden_index("adv")
    fa = _reads_fa(tmp_path)
    p = subprocess.run([EXE, "-f", "-x", base, "-U", fa, "--tab-fmt-cols", "readID,score,hitLength", "--kreport-file", str(tmp_path / "k"),
                        "-S", str(tmp_path / "o.tsv")],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    assert p.returncode == 1 and b"--kreport-file needs" in p.stderr


# ----------------------------------------------------------------------------- host formatter
IUPAC = b"RYKMSWBDHV"


def decorate(rng, rs, fasta):
    """Spellings the readers map to codes: lower case, '.' (FASTQ: N; FASTA: not a base), IUPAC letters, N runs that fail
    the N filter, very short reads that trims empty."""
    out = []
    for n, s in rs:
        s = bytearray(s)
        r = rng.random()
        if r < 0.1:
            s = bytearray(bytes(s).lower())
        elif r < 0.2 and len(s) > 8:
            s[3] = ord(".")
        elif r < 0.3 and len(s) > 8:
            s[2] = rng.choice(IUPAC); s[6] = rng.choice(IUPAC.lower())
        elif r < 0.38:
            for _ in range(max(1, len(s) // 4)):
                s[rng.randrange(len(s))] = ord("N")
        elif r < 0.45:
            s = s[:rng.randrange(1, 9)]
        out.append((n, bytes(s)))
    return out


def write_reads(path, rs, fasta, rng):
    with open(path, "wb") as f:
        for i, (n, s) in enumerate(rs):
            name = n + (b" desc" if i % 7 == 3 else b"") + (b"/1" if i % 5 == 2 else b"")
            if fasta:
                f.write(b">" + name + b"\n" + s + b"\n")
            else:
                nq = len(s) + (1 if rng.random() < 0.2 else 0)                 # one spare quality value
                f.write(b"@" + name + b"\n" + s + b"\n+\n" + bytes(rng.randrange(33, 127) for _ in range(nq)) + b"\n")


def random_cols(rng):
    r = rng.random()
    if r < 0.15:
        return DEFAULT
    if r < 0.35:
        return WRAPPER
    return ",".join(rng.choice(NAMES) for _ in range(rng.randrange(1, 12)))


def test_host_formatter_reproduces_reference_columns(tmp_path):
    util.ensure_oracle()
    base = util.golden_index("adv")
    lib = C.CDLL(util.PRODUCT_LIB)
    reads = clean_reads()
    o = util.Oracle(base)
    from test_host_path import dump_reads
    for case in range(200):
        rng = random.Random(51000 + case)
        oi = rng.randrange(len(API_OPTS))
        kw, cli = API_OPTS[oi], CLI_OPTS[oi]
        fasta, paired = rng.random() < 0.5, rng.random() < 0.4
        trims = rng.choice([(0, 0), (0, 0), (2, 0), (0, 4), (3, 5)])
        seed = rng.choice([0, 0, 7, 12345])
        cols = random_cols(rng)
        rs = decorate(rng, make_reads(rng, reads), fasta)
        p1, p2 = str(tmp_path / "a.txt"), str(tmp_path / "b.txt")
        if paired:
            rs2 = decorate(rng, make_reads(rng, reads), fasta)[:len(rs)]; rs = rs[:len(rs2)]
            rs = [(n, x if len(x) >= 10 else x + b"ACGTACGTAC") for n, x in rs]     # the reference crashes on a pair whose first mate trims to nothing
            write_reads(p2, rs2, fasta, rng)
        write_reads(p1, rs, fasta, rng)
        m1 = dump_reads(lib, p1, fasta, trims, tmp_path)
        bt = util.Batch(m1, dump_reads(lib, p2, fasta, trims, tmp_path)) if paired else util.Batch(m1)
        on, orec, _ = o.classify(bt, util.make_oparams(**kw))
        rec_off = np.concatenate([[0], np.cumsum(on)]).astype(np.uint32)
        recs = np.ascontiguousarray(orec)
        tsv, rep = str(tmp_path / "p.tsv"), str(tmp_path / "p.rep")
        rc = lib.cfb_test_host_path_cols(base.encode(), p1.encode(), p2.encode() if paired else None, C.c_int(1 if fasta else 0), C.c_int(kw.get("k", 5)),
                                         C.c_uint32(seed), C.c_int(trims[0]), C.c_int(trims[1]), rec_off.ctypes.data_as(C.POINTER(C.c_uint32)),
                                         recs.ctypes.data_as(C.c_void_p), C.c_uint64(len(on)), cols.encode(), tsv.encode(), rep.encode(), None)
        assert rc == 0, (case, rc)
        args = ["-f" if fasta else "-q", "-x", base, "--seed", str(seed), "-5", str(trims[0]), "-3", str(trims[1]), "--tab-fmt-cols", cols] + cli + (["-1", p1, "-2", p2] if paired else ["-U", p1])
        with open(tsv, "rb") as f, open(rep, "rb") as g:
            got = (f.read(), g.read())
        want = util_cols.reference("tab_cols/host/%d" % case, lambda: util.run_cli(util.REF_CLASS, args, str(tmp_path / "r.tsv"), str(tmp_path / "r.rep")))
        util.assert_matches(got, want, case, cols, kw, fasta, paired, trims, seed)
    o.close()


# ----------------------------------------------------------------------------- the wrapper
def wrapper_inputs(tmp, fasta, paired):
    """Small SE/PE inputs for the wrapper cases, from the golden index's reads (some unclassifiable)."""
    rng = random.Random(7 + 2 * fasta + paired)
    reads = clean_reads()
    rs = decorate(rng, make_reads(rng, reads) + make_reads(rng, reads), fasta)
    ext = "fa" if fasta else "fq"
    p1, p2 = str(tmp / ("w1." + ext)), str(tmp / ("w2." + ext))
    if paired:
        rs2 = decorate(rng, make_reads(rng, reads) + make_reads(rng, reads), fasta)[:len(rs)]; rs = rs[:len(rs2)]
        write_reads(p2, [(n, s if len(s) else b"A") for n, s in rs2], fasta, rng)
    write_reads(p1, [(n, s if len(s) else b"A") for n, s in rs], fasta, rng)
    return (["-1", p1, "-2", p2] if paired else ["-U", p1]), p1, p2


WRAPPER_CASES = [(fasta, paired, mode) for fasta in (0, 1) for paired in (0, 1) for mode in sorted(WRAPPER_MODES)
                 if not (paired and mode in ("un", "al")) and not (not paired and mode.endswith("conc"))]


def wrapper_case(tmp, fasta, paired):
    base = util.golden_index("adv")
    io, _, _ = wrapper_inputs(tmp, fasta, paired)
    return base, ["-f" if fasta else "-q", "-x", base] + io


@pytest.mark.parametrize("fasta,paired,mode", WRAPPER_CASES)
def test_wrapper_split_restatement(fasta, paired, mode, tmp_path):
    """The restated split, applied to the reference binary's stdout under the wrapper's command line, gives the files
    the real wrapper wrote (recorded digests; re-checked against the wrapper itself where the reference tree is present)."""
    util.ensure_oracle()
    base, args = wrapper_case(tmp_path, fasta, paired)
    key = "tab_cols/wrapper/%d%d%s" % (fasta, paired, mode)
    cmd = ["--wrapper", "basic-0"] + args + wrapper_cols(mode) + ["--passthrough", "--report-file", str(tmp_path / "rr")]
    want_out = util_cols.reference(key + "/stdout", lambda: subprocess.run([util.REF_CLASS] + cmd, stdout=subprocess.PIPE, check=True).stdout)
    want_files = util_cols.reference(key + "/files", lambda: run_real_wrapper(tmp_path, args, mode))
    if not util.have_ref():
        pytest.skip("the reference binary is not built here; the GPU tests apply the split to the product's stdout")
    stdout = subprocess.run([util.REF_CLASS] + cmd, stdout=subprocess.PIPE, check=True).stdout
    util.assert_matches(stdout, want_out)
    util.assert_matches(split_for(mode, stdout), want_files, mode)
