"""--n-ceil on the GPU: centrifuge-class under every test ceiling against the reference binary's recorded outputs, through
the device text operator (no fallback on strict input) and the record-level reader; the C ABI's cfb_ctx_set_n_ceil;
N-dense reads under L,0,1 reaching their full hit lists; --ignore-quals / --nofw / --norc; and the device's log and
sqrt against the host's over every mate length."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import util
import util_nceil as U

CLI = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
STATS = re.compile(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units")
LONG = re.compile(r"long units: (\d+) \((\d+) bases\)")


@pytest.fixture(scope="module")
def inputs():
    return U.write_inputs(os.path.join(util.CACHE, "n_ceil_inputs"))


def _run(tmp, args, stats=False):
    import subprocess
    env = dict(os.environ, CFB_TEXT_STATS="1") if stats else None
    p = subprocess.run([CLI] + args + ["-S", os.path.join(str(tmp), "o.tsv"), "--report-file", os.path.join(str(tmp), "o.rep")],
                       stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=env)
    assert p.returncode == 0, p.stderr.decode()[-2000:]
    with open(os.path.join(str(tmp), "o.tsv"), "rb") as f, open(os.path.join(str(tmp), "o.rep"), "rb") as g:
        return (f.read(), g.read()), p.stderr.decode()


def _want(adv_base, tmp, name, args, extra, key):
    return U.reference(key, lambda: U.run_cli(util.REF_CLASS, ["-x", adv_base] + args + extra, tmp))


@pytest.mark.gpu
@pytest.mark.parametrize("spec", U.CEILS, ids=U.ceil_key)
@pytest.mark.parametrize("name", ["se", "fa", "gz", "fagz", "pe", "empty"])
def test_cli_matches_reference(adv_base, inputs, tmp_path, spec, name):
    """TSV, report and Kraken-style report equal the reference's, through the text operator and with --host-parse"""
    args = inputs[name]
    ref = U.REF_OF.get(name, name)
    want = _want(adv_base, tmp_path, ref, inputs[ref], U.ceil_args(spec), "%s/%s" % (ref, U.ceil_key(spec)))
    want_kr = U.reference("kreport/%s/%s" % (ref, U.ceil_key(spec)), lambda: U.ref_kreport(adv_base, inputs[ref] + U.ceil_args(spec), tmp_path))
    if util.RECORD:
        return
    kr = os.path.join(str(tmp_path), "o.kreport")
    got, err = _run(tmp_path, ["-x", adv_base, "--kreport-file", kr] + args + U.ceil_args(spec), stats=True)
    util.assert_matches(got, want, name, spec)
    with open(kr, "rb") as f:
        util.assert_matches(f.read(), want_kr, name, spec, "kreport")
    m = STATS.search(err)
    assert m, err
    if name in ("se", "pe"):             # strict FASTQ: every unit through the device tokeniser
        assert int(m.group(3)) == 0 and int(m.group(4)) == 0, err
    if name in ("se", "pe", "empty"):
        got, _ = _run(tmp_path, ["-x", adv_base, "--host-parse"] + args + U.ceil_args(spec))
        util.assert_matches(got, want, name, spec, "host-parse")


@pytest.mark.gpu
@pytest.mark.parametrize("spec", ["L,0,1", "G,0,3", "C,0"])
@pytest.mark.parametrize("extra", [["-k", "1"], ["-k", "40"], ["-k", "5", "--host-taxids", "9606,1"]], ids=["k1", "k40", "host"])
@pytest.mark.parametrize("name", ["se", "pe"])
def test_cli_k_and_host_taxids(adv_base, inputs, tmp_path, spec, extra, name):
    args = inputs[name]
    key = "%s/%s/%s" % (name, U.ceil_key(spec), "_".join(extra))
    want = _want(adv_base, tmp_path, name, args, extra + U.ceil_args(spec), key)
    if util.RECORD:
        return
    got, _ = _run(tmp_path, ["-x", adv_base] + extra + args + U.ceil_args(spec))
    util.assert_matches(got, want, spec, extra)
    got, _ = _run(tmp_path, ["-x", adv_base, "--host-parse"] + extra + args + U.ceil_args(spec))
    util.assert_matches(got, want, spec, extra, "host-parse")


@pytest.mark.gpu
def test_cli_two_devices(adv_base, inputs, tmp_path):
    want = _want(adv_base, tmp_path, "pe", inputs["pe"], ["--n-ceil", "L,0,1"], "pe/c[L,0,1]")
    if util.RECORD:
        return
    from centrifuge_b200 import capi
    if capi.lib().cfb_device_count() < 2:
        pytest.skip("one GPU")
    got, _ = _run(tmp_path, ["-x", adv_base, "--devices", "0,1"] + inputs["pe"] + ["--n-ceil", "L,0,1"])
    util.assert_matches(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", U.QUIRK_FLAGS, ids=lambda f: "+".join(x.strip("-") for x in f))
def test_quirk_flags_change_nothing(adv_base, inputs, tmp_path, flags):
    args = inputs["se"]
    want = _want(adv_base, tmp_path, "se", args, flags, "se/default/" + "+".join(flags))
    if util.RECORD:
        return
    assert want == U.reference("se/default", None)
    got, _ = _run(tmp_path, ["-x", adv_base] + flags + args)
    util.assert_matches(got, want, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("spec", ["L,0,1", "S,1,2", "G,0,3", "C,-3"])
def test_capi_text_equals_classify_with_host_flags(adv_base, spec):
    """cfb_ctx_set_n_ceil + cfb_text_submit gives the rows of cfb_classify_batch fed with flags computed on the host"""
    from centrifuge_b200 import capi
    singles, _, _ = U.make_reads()
    reads = [(n, s) for n, s in singles if len(s) > 0 and len(s) <= 60000]
    f = U.PARSED[spec]
    text = U.fastq(reads)
    ix = capi.Index(adv_base, 0)
    ctx = capi.Context(ix)
    try:
        ctx.set_n_ceil(f[0], f[1], f[2])
        ctx.text_submit(0, np.frombuffer(text, dtype=np.uint8).copy(), None, len(reads), fasta=False)
        r = ctx.text_wait(0)
        assert not r["irregular"]
        b = util.Batch([np.frombuffer(s.encode(), dtype=np.uint8) for _, s in reads])
        flags = np.array([1 if U.passes(f, s) else 0 for _, s in reads], dtype=np.uint8)
        off, recs = ctx.classify(capi.make_batch(b.bases, b.off1, b.len1, None, None, flags))
        o = util.Oracle(adv_base)
        on, orec, _ = o.classify(b_with(b, flags), util.make_oparams())
        o.close()
        assert np.array_equal(np.diff(off.astype(np.int64)), on.astype(np.int64))
        for k in ("taxid", "score", "hitlen", "uid"):
            assert np.array_equal(orec[k], recs[k]), k
        # a read the ceiling filters gets one "unclassified" row; one it passes gets rows only if it has records
        rows = {}
        for row in r["tsv"].split(b"\n"):
            if row:
                rows.setdefault(row.split(b"\t")[0].decode(), []).append(row.split(b"\t")[1])
        nrec = np.diff(off.astype(np.int64))
        for i, (name, _) in enumerate(reads):
            if flags[i] == 0 or nrec[i] == 0:
                assert rows[name] == [b"unclassified"], name
            else:
                assert b"unclassified" not in rows[name], name
    finally:
        ctx.close()
        ix.close()


def b_with(b, flags):
    b.flags = flags
    return b


@pytest.mark.gpu
def test_ndense_reads_reach_full_hit_lists(adv_base, inputs, tmp_path):
    """under L,0,1 reads with an N every 2nd or 3rd base pass, and their records equal the oracle's (no truncated list);
    the context's ceiling sizes the batch's hit lists (nceil_full_cap): the same batch on a context left at the default
    ceiling overflows them and runs its search again, with the same records"""
    from centrifuge_b200 import capi
    singles, _, _ = U.make_reads()
    f = U.PARSED["L,0,1"]
    reads = [s for _, s in singles if len(s) >= 2 and s.count("N") + s.count(".") > 0.3 * len(s)]
    assert len(reads) > 20
    b = util.Batch([np.frombuffer(s.replace(".", "N").encode(), dtype=np.uint8) for s in reads])
    flags = np.array([1 if U.passes(f, s) else 0 for s in reads], dtype=np.uint8)
    assert flags.all()
    ix = capi.Index(adv_base, 0)
    ctx = capi.Context(ix)
    try:
        ctx.set_n_ceil(f[0], f[1], f[2])
        off, recs = ctx.classify(capi.make_batch(b.bases, b.off1, b.len1, None, None, flags))
        o = util.Oracle(adv_base)
        on, orec, _ = o.classify(b_with(b, flags), util.make_oparams())
        o.close()
        assert np.array_equal(np.diff(off.astype(np.int64)), on.astype(np.int64))
        for k in ("taxid", "score", "hitlen", "uid"):
            assert np.array_equal(orec[k], recs[k]), k
        ctx2 = capi.Context(ix)
        try:
            off2, recs2 = ctx2.classify(capi.make_batch(b.bases, b.off1, b.len1, None, None, flags))
            assert np.array_equal(off, off2) and np.array_equal(recs, recs2)
            assert ctx.launches() < ctx2.launches(), (ctx.launches(), ctx2.launches())
        finally:
            ctx2.close()
    finally:
        ctx.close()
        ix.close()
    _, err = _run(tmp_path, ["-x", adv_base] + inputs["se"] + ["--n-ceil", "L,0,1"], stats=True)
    m = LONG.search(err)
    assert m and int(m.group(1)) == 2 and int(m.group(2)) == 2 * 60001, err        # the two 60 001-base reads, N-dense one included


@pytest.mark.gpu
def test_device_log_and_sqrt_equal_host_for_every_length():
    """G and S ceilings: the device's sqrt of every mate length 1 .. 2^31 - 1 is the host's, bit for bit, and its log at
    most one unit in the last place off (where that can move a ceiling the read goes to the host reader)"""
    from centrifuge_b200 import capi
    nl, nf, ns, first = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = capi.lib().cfb_test_log_sqrt(0, C.c_uint64(1), C.c_uint64(2 ** 31), C.byref(nl), C.byref(nf), C.byref(ns), C.byref(first))
    assert rc == 0
    assert ns.value == 0                  # sqrt: bit for bit (both correctly rounded)
    assert nf.value == 0, "log more than one unit in the last place off at %d lengths" % nf.value   # what k_tok_bases' check assumes
    print("device log differs from the host's in the last bit at %d of 2^31 - 1 lengths (the first %d)" % (nl.value, first.value))
