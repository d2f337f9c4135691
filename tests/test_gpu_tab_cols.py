"""--tab-fmt-cols on the device: the text operator's formatter prints every column list with the reference's bytes,
strict input stays on the device, irregular input, --host-parse and several devices give the same bytes, the
`centrifuge` wrapper's exact command line works end to end, and cfb_ctx_set_columns gives the CLI's rows."""
import os
import subprocess

import numpy as np
import pytest

import util
import util_cols
from test_gpu_text import decorate, run_ours, write_fq, syn  # noqa: F401  (syn is a fixture)
from test_tab_cols import DEFAULT, NAMES, WRAPPER, WRAPPER_CASES, run_real_wrapper, split_for, wrapper_case, wrapper_cols

pytestmark = pytest.mark.gpu

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
LISTS = [WRAPPER, "readID,taxName,taxRank,SEQ1,QUAL1,SEQ2,QUAL2,CIGAR,FLAG,TLEN,RNAME", ",".join(NAMES), DEFAULT + ",taxName,readSeq,readID"]


def run_ref(key, args, tmp, tag):
    """digest of the reference's (TSV, report) for these arguments"""
    return util_cols.reference("gpu_text/" + key, lambda: util.run_cli(util.REF_CLASS, args, str(tmp / (tag + ".tsv")), str(tmp / (tag + ".rep"))))


def se_input(syn, tmp):
    base, seqs = syn
    rng = np.random.default_rng(21)
    reads = (util.synth.sample_reads(seqs, 1500, 60, seed=61, lens=(1, 120)) + util.synth.sample_reads(seqs, 1500, 150, seed=62, lens=(100, 300))
             + util.synth.sample_reads(seqs, 200, 500, seed=63, lens=(300, 900)))
    reads = decorate(reads, rng)
    fq = str(tmp / "c.fq")
    write_fq(fq, reads, rng)
    return base, fq, len(reads)


def pe_input(syn, tmp):
    base, seqs = syn
    rng = np.random.default_rng(22)
    prs = util.synth.sample_pairs(seqs, 3000, 125, seed=71)
    r1 = decorate([(n, x) for n, x, _ in prs], rng)
    r2 = [(n + "/2", y[: max(1, len(y) - (i % 40))]) for i, (n, _, y) in enumerate(prs)]
    f1, f2 = str(tmp / "c_1.fq"), str(tmp / "c_2.fq")
    write_fq(f1, r1, rng); write_fq(f2, r2, rng)
    return base, f1, f2, len(prs)


@pytest.mark.parametrize("li", range(len(LISTS)))
def test_columns_on_device_match_reference(li, syn, tmp_path):
    cols = LISTS[li]
    base, fq, n = se_input(syn, tmp_path)
    for extra in ([], ["-5", "3", "-3", "7"], ["-k", "9", "--min-hitlen", "15"]):
        args = ["-q", "-x", base, "-U", fq, "--tab-fmt-cols", cols] + extra
        want = run_ref("tab_cols/se/%d/%s" % (li, " ".join(extra)), args, tmp_path, "ref")
        got, st = run_ours(args, tmp_path, "our", block=100000)
        util.assert_matches(got, want, cols, extra)
        assert st["fallbacks"] == 0 and st["host"] == 0 and st["text"] == n, st
    base, f1, f2, n = pe_input(syn, tmp_path)
    for extra in ([], ["-3", "100"], ["-k", "2"]):
        args = ["-q", "-x", base, "-1", f1, "-2", f2, "--tab-fmt-cols", cols] + extra
        want = run_ref("tab_cols/pe/%d/%s" % (li, " ".join(extra)), args, tmp_path, "ref")
        got, st = run_ours(args, tmp_path, "our", block=150000)
        util.assert_matches(got, want, cols, extra)
        assert st["fallbacks"] == 0 and st["host"] == 0 and st["text"] == n, st
        got2, st2 = run_ours(args + ["--host-parse"], tmp_path, "host")
        assert got2 == got and st2["text"] == 0


def test_fasta_columns_on_device(syn, tmp_path):
    base, seqs = syn
    rng = np.random.default_rng(23)
    reads = decorate(util.synth.sample_reads(seqs, 3000, 100, seed=65, lens=(20, 200)), rng)
    reads = [(n, np.frombuffer(a.tobytes().replace(b".", b"N"), dtype=np.uint8)) for n, a in reads]
    fa = str(tmp_path / "c.fa")
    with open(fa, "wb") as f:
        for n, a in reads:
            f.write(b">" + n.encode() + b"\n" + a.tobytes() + b"\n")
    for key, args in (("fasta_se", ["-f", "-x", base, "-U", fa]), ("fasta_pe", ["-f", "-x", base, "-1", fa, "-2", fa, "-5", "2"])):
        args = args + ["--tab-fmt-cols", WRAPPER + ",SEQ2,QUAL2"]
        got, st = run_ours(args, tmp_path, "our", block=50000)
        util.assert_matches(got, run_ref("tab_cols/" + key, args, tmp_path, "ref"))
        assert st["fallbacks"] == 0 and st["text"] == len(reads), st


def test_irregular_input_falls_back_with_the_same_bytes(syn, tmp_path):
    base, seqs = syn
    reads = util.synth.sample_reads(seqs, 3000, 100, seed=21, lens=(40, 140))
    fq = str(tmp_path / "r.fq")
    with open(fq, "wb") as f:
        for i, (name, a) in enumerate(reads):
            rec = b"@" + name.encode() + b"\n" + a.tobytes() + b"\n+\n" + b"F" * len(a) + b"\n"
            f.write(rec.replace(b"\n", b"\r\n") if i == 2000 else rec)
    args = ["-q", "-x", base, "-U", fq, "--tab-fmt-cols", WRAPPER]
    got, st = run_ours(args, tmp_path, "our", block=60000)
    util.assert_matches(got, run_ref("tab_cols/irregular", args, tmp_path, "ref"))
    assert st["fallbacks"] == 1 and st["text"] > 1000 and st["host"] > 900, st


def test_several_devices_give_one_device_bytes(syn, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    base, fq, n = se_input(syn, tmp_path)
    args = ["-q", "-x", base, "-U", fq, "--tab-fmt-cols", LISTS[1]]
    one, _ = run_ours(args, tmp_path, "one", block=100000)
    two, st = run_ours(args + ["--devices", "0-1"], tmp_path, "two", block=100000)
    assert one == two and st["fallbacks"] == 0


def test_defaults_unchanged(syn, tmp_path):
    base, fq, n = se_input(syn, tmp_path)
    plain, _ = run_ours(["-q", "-x", base, "-U", fq], tmp_path, "plain", block=100000)
    passthru, _ = run_ours(["-q", "-x", base, "-U", fq, "--passthrough"], tmp_path, "pt", block=100000)
    assert passthru == plain
    kr_a, kr_b = str(tmp_path / "a.kr"), str(tmp_path / "b.kr")
    run_ours(["-q", "-x", base, "-U", fq, "--kreport-file", kr_a], tmp_path, "ka", block=100000)
    run_ours(["-q", "-x", base, "-U", fq, "--kreport-file", kr_b, "--tab-fmt-cols", "numMatches,readSeq," + WRAPPER], tmp_path, "kb", block=100000)
    assert open(kr_a, "rb").read() == open(kr_b, "rb").read() and os.path.getsize(kr_a) > 0
    p = subprocess.run([EXE, "-q", "-x", base, "-U", fq, "--tab-fmt-cols", "readID,score,hitLength", "--kreport-file", kr_a, "-S", str(tmp_path / "x.tsv")],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    assert p.returncode == 1 and b"--kreport-file needs" in p.stderr


@pytest.mark.parametrize("fasta,paired,mode", WRAPPER_CASES)
def test_wrapper_command_line(fasta, paired, mode, tmp_path):
    """centrifuge-class as the `centrifuge` script runs it for --un / --al / --un-conc / --al-conc / --no-unal: rows on
    stdout, no -S; the script's split of them gives the files the real script wrote with the reference binary."""
    base, args = wrapper_case(tmp_path, fasta, paired)
    key = "tab_cols/wrapper/%d%d%s" % (fasta, paired, mode)
    cmd = ["--wrapper", "basic-0"] + args + wrapper_cols(mode) + ["--passthrough", "--report-file", str(tmp_path / "rr")]
    p = subprocess.run([EXE] + cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1"))
    assert p.returncode == 0, p.stderr.decode()
    util.assert_matches(p.stdout, util_cols.reference(key + "/stdout", lambda: subprocess.run([util.REF_CLASS] + cmd, stdout=subprocess.PIPE, check=True).stdout))
    util.assert_matches(split_for(mode, p.stdout), util_cols.reference(key + "/files", lambda: run_real_wrapper(tmp_path, args, mode)), mode)


def test_capi_columns_match_cli(syn, tmp_path):
    from centrifuge_b200 import capi
    base, fq, n = se_input(syn, tmp_path)
    text = open(fq, "rb").read()
    ix = capi.Index(base, 0)
    ctx = capi.Context(ix)
    try:
        for cols in (WRAPPER, LISTS[1], None):
            args = ["-q", "-x", base, "-U", fq] + (["--tab-fmt-cols", cols] if cols else [])
            (tsv, _), st = run_ours(args, tmp_path, "cli")
            assert st["spans"] == 1 and st["fallbacks"] == 0
            ctx.set_columns(cols)
            ctx.text_submit(0, np.frombuffer(text, dtype=np.uint8).copy(), None, n, maxlen_hint=900)
            r = ctx.text_wait(0, discard=True)
            assert not r["irregular"] and r["tsv"] == tsv.split(b"\n", 1)[1], cols
        with pytest.raises(capi.CfbError, match="Column definition bogus invalid."):
            ctx.set_columns("readID,bogus")
        with pytest.raises(capi.CfbError, match="error -1"):
            ctx.set_columns("")
    finally:
        ctx.close(); ix.close()
