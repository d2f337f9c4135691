"""Quality encodings on the GPU: centrifuge-class under every encoding option against the reference binary's recorded
outputs (TSV, report, Kraken-style report) through the device text operator (no fallback on strict input) and the
record-level reader; the refusals; tie selection by the per-read seed on the tie-rich index under --host-taxids; the C
ABI's cfb_ctx_set_quals; and several devices."""
import os
import re
import subprocess

import numpy as np
import pytest

import util
import util_nceil
import util_quals as U
import util_ties

CLI = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
STATS = re.compile(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units")


def _dir():
    return os.path.join(util.CACHE, "quals_inputs")


def _run(tmp, args, stats=False):
    env = dict(os.environ, CFB_TEXT_STATS="1") if stats else None
    p = subprocess.run([CLI] + args + ["-S", os.path.join(str(tmp), "o.tsv"), "--report-file", os.path.join(str(tmp), "o.rep")],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=env)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    with open(os.path.join(str(tmp), "o.tsv"), "rb") as f, open(os.path.join(str(tmp), "o.rep"), "rb") as g:
        return (f.read(), g.read()), p.stderr.decode()


CLI_CASES = [(m, "se") for m in U.MODES] + [(m, w) for m in U.MAIN for w in ("pe", "gz", "trim", "long", "fa")] + \
            [(m, w) for m in U.MAIN if U.is_int(m) for w in ("quirks", "line4096")]


@pytest.mark.gpu
@pytest.mark.parametrize("cols", ["default", "quals"])
@pytest.mark.parametrize("mode,which", CLI_CASES, ids=["%s-%s" % c for c in CLI_CASES])
def test_cli_matches_reference(adv_base, tmp_path, mode, which, cols):
    """TSV and report (and with the default columns the Kraken-style report) equal the reference's, through the text
    operator and with --host-parse; an input the reference refuses is refused with its messages"""
    inputs = U.inputs(_dir(), mode)
    ref = U.REF_OF.get(which, which)
    extra = U.MODES[mode][0] + ([] if cols == "default" else ["--tab-fmt-cols", U.QCOLS])
    key = "cli/%s/%s/%s" % (ref, mode, cols)
    refused = U.is_int(mode) and which == "long"           # the 4200-byte integer line: the reference stops with an error
    if refused:
        want = U.reference(key, lambda: U.run_ref_error(util.REF_CLASS, adv_base, extra + inputs[ref], tmp_path))
    else:
        want = U.reference(key, lambda: util_nceil.run_cli(util.REF_CLASS, ["-x", adv_base] + extra + inputs[ref], tmp_path))
    want_kr = None
    if cols == "default" and not refused:
        want_kr = U.reference("kreport/" + key, lambda: util_nceil.ref_kreport(adv_base, extra + inputs[ref], tmp_path))
    if util.RECORD:
        return
    for host in (False, True):
        args = ["-x", adv_base] + (["--host-parse"] if host else []) + extra + inputs[which]
        if refused:
            got = U.run_ref_error(CLI, adv_base, args[2:], tmp_path)
            util.assert_matches((got[0], got[1], b""), want, mode, which, host)
            continue
        kr = os.path.join(str(tmp_path), "o.kreport")
        got, err = _run(tmp_path, args + (["--kreport-file", kr] if want_kr else []), stats=True)
        util.assert_matches(got, want, mode, which, cols, host)
        if want_kr:
            with open(kr, "rb") as f:
                util.assert_matches(f.read(), want_kr, mode, which, "kreport", host)
        m = STATS.search(err)
        assert m, err
        if not host and which in ("se", "pe", "gz") and U.MODES[mode][1] != "p33":
            assert int(m.group(3)) == 0 and int(m.group(4)) == 0, err          # strict input: every unit on the device
        if not host and which == "line4096":
            assert int(m.group(3)) >= 1, err                                    # lines of 4095 bytes and more: the host decides


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(U.ERRORS))
def test_cli_refusals_match_reference(adv_base, tmp_path, case):
    mode, trims = U.ERRORS[case]
    path = U.write(os.path.join(str(tmp_path), "bad.fq"), U.fastq(U.error_records(case)))
    args = U.MODES[mode][0] + ["-5", str(trims[0]), "-3", str(trims[1]), "-U", path]
    want = U.reference("error/" + case, lambda: U.run_ref_error(util.REF_CLASS, adv_base, args, tmp_path))
    if util.RECORD:
        return
    for host in ([], ["--host-parse"]):
        got = U.run_ref_error(CLI, adv_base, host + args, tmp_path)
        assert got[0] and got[1]
        util.assert_matches((got[0], got[1], b""), want, case, host)


def _ties_reads(kind):
    import random
    rng = random.Random(3)
    out = []
    for n, a in util_ties.single_reads():
        s = a.tobytes() if hasattr(a, "tobytes") else bytes(a)
        lo, hi = (10, 60) if kind in ("sol", "intsol") else (0, 60)
        out.append((n.encode(), s, U.render(kind, [rng.randint(lo, hi) for _ in s])))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("mode", U.MAIN)
def test_seeds_pick_the_reference_rows(tmp_path, mode, k):
    """more than -k records tie under --host-taxids: the per-read seed, which hashes the converted qualities, picks the rows"""
    base = util.golden_index("ties_plain")              # the committed tie-rich index (util_ties.index without re-recording it)
    kind = U.MODES[mode][1]
    fq = U.write(os.path.join(_dir(), "ties.%s.fq" % kind), U.fastq(_ties_reads(kind)))
    args = U.MODES[mode][0] + ["-k", str(k), "--host-taxids", ",".join(map(str, util_ties.HOST)), "--tab-fmt-cols", U.QCOLS + ",taxID,score", "-U", fq]
    want = U.reference("ties/%s/k%d" % (mode, k), lambda: util_nceil.run_cli(util.REF_CLASS, ["-x", base] + args, tmp_path))
    if util.RECORD:
        return
    for host in ([], ["--host-parse"]):
        got, _ = _run(tmp_path, ["-x", base] + host + args)
        util.assert_matches(got, want, mode, k, host)


@pytest.mark.gpu
def test_capi_renderings_give_the_phred33_rows(adv_base):
    """cfb_ctx_set_quals + cfb_text_submit on phred64, Solexa-range and integer renderings of one phred33 span give the
    phred33 span's rows byte for byte, quality columns included"""
    from centrifuge_b200 import capi
    import random
    rng = random.Random(8)
    src = U._adv_reads()[:3000]
    vals = [[rng.randint(10, 60) for _ in s] for s in src]           # >= 10: Solexa and Phred values coincide
    names = [("q%d" % i).encode() for i in range(len(src))]
    span = {k: U.fastq([(n, s, U.render(k, v)) for n, s, v in zip(names, src, vals)]) for k in ("p33", "p64", "sol", "int")}
    enc = {"p33": {}, "p64": dict(phred64=True), "sol": dict(solexa=True), "int": dict(integer=True)}
    ix = capi.Index(adv_base, 0)
    ctx = capi.Context(ix)
    try:
        ctx.set_columns("readID,readSeq,readQual,QUAL,taxID,score")
        rows = {}
        for k in ("p33", "p64", "sol", "int", "p33"):
            ctx.set_quals(**enc[k])
            ctx.text_submit(0, np.frombuffer(span[k], dtype=np.uint8).copy(), None, len(src))
            r = ctx.text_wait(0)
            assert not r["irregular"], k
            rows.setdefault(k, r["tsv"])
            assert r["tsv"] == rows["p33"], k
        with pytest.raises(capi.CfbError):
            ctx.set_quals(solexa=2)
    finally:
        ctx.close()
        ix.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["int-quals", "solexa-quals"])
def test_cli_two_devices(adv_base, tmp_path, mode):
    inputs = U.inputs(_dir(), mode)
    extra = U.MODES[mode][0] + ["--tab-fmt-cols", U.QCOLS]
    want = U.reference("cli/pe/%s/quals" % mode, lambda: util_nceil.run_cli(util.REF_CLASS, ["-x", adv_base] + extra + inputs["pe"], tmp_path))
    if util.RECORD:
        return
    from centrifuge_b200 import capi
    if capi.lib().cfb_device_count() < 2:
        pytest.skip("one GPU")
    got, _ = _run(tmp_path, ["-x", adv_base, "--devices", "0,1"] + extra + inputs["pe"])
    util.assert_matches(got, want, mode)
