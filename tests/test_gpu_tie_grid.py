"""GPU: tie selection and the taxonomy reduction across -k 1 to 64, on the tie-rich fixture (util_ties.py) with its NCBI-shaped
lineages, against the oracle and the reference.

- Through the C ABI, every (build, layout) runs -k 1 to 64 with the default options, a host set holding more than 32 tied
  sequences, an exclude set, --classification-rank genus and family, --no-traverse and --min-hitlen 15, single-end and paired,
  and compares every record with the oracle's.  The counting instantiation of k_score shows that the grid reaches tree
  reductions over several rank rounds at -k >= 2 and warps whose hit maps live in the global scratch.
- centrifuge-class writes the reference's TSV, report and Kraken-style report (recorded digests) at -k 2 to 64 through the text
  operator and through the record-level reader (--host-parse), with the reader its CFB_TEXT_STATS line reports: the text
  operator alone up to -k 32 unless a unit has more than 32 records (only under --host-taxids), the record-level reader for
  the rest of the file after such a unit, and the record-level reader alone from -k 33.
- The per-taxon counters: the text operator's equal a fold of its own rows, and the record-level path's equal a fold of the
  records that counts the first k tied best records of a unit in record order."""
import concurrent.futures
import os
import re
import subprocess

import numpy as np
import pytest

import util
import util_ties as T
from test_gpu_parity import assert_same, to_cbatch
from test_tie_grid_host import oracle_records, reference_outputs, units

pytestmark = pytest.mark.gpu

LAYOUTS = {"default": {}, "compact": {"CFB_RANK16": "0"}, "kmer_at_ftab": {"CFB_FTABK": "FC"}}
KNOBS = ("CFB_RANK16", "CFB_FTABK", "CFB_FTABD", "CFB_RESOLVE_TABLE", "CFB_WALK8", "CFB_WALK8_ROWS", "CFB_KEEP_SHORT", "CFB_COUNT",
         "CFB_HBM_HEADROOM_GB", "CFB_REGEN_SLOTS", "CFB_REGEN_STATS", "CFB_ROWS_CAP")
EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")


def capi():
    from centrifuge_b200 import capi as m
    return m


def set_env(monkeypatch, env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def params(k, case):
    return capi().make_params(k=k, **T.OPTIONS[case])


def classify(ctx, b):
    off, recs = ctx.classify(to_cbatch(b))
    return np.diff(off.astype(np.int64)).astype(np.uint32), recs


@pytest.mark.parametrize("build", T.BUILDS)
def test_project_builder_writes_the_committed_index(build):
    T.project_build(build)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("build", T.BUILDS)
def test_tie_grid_matches_oracle(build, layout, monkeypatch):
    base = T.index(build)              # before the threads: they all read it
    keys = [(build, rs, k, case) for rs in ("se", "pe") for k in T.K_GRID for case in T.OPTIONS]
    with concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(lambda a: oracle_records(*a), keys))
    m = capi()
    set_env(monkeypatch, {})
    ix = m.Index(base, 0)
    fc = ix.info.ftab_chars
    ix.close()
    set_env(monkeypatch, {k: v.replace("FC", str(fc)) for k, v in LAYOUTS[layout].items()})
    ix = m.Index(base, 0)
    tb = ix.tables()
    assert (tb["rank16_bytes"] == 0) == (layout == "compact"), tb
    assert layout != "kmer_at_ftab" or tb["ftabk_chars"] == fc, tb
    bad = []
    try:
        for _, rs, k, case in keys:
            ctx = m.Context(ix, params(k, case))
            gn, grec = classify(ctx, T.batches()[rs])
            ctx.close()
            try:
                assert_same(*oracle_records(build, rs, k, case), gn, grec)
            except AssertionError as e:
                bad.append("%s k %d %s: %s" % (rs, k, case, e))
    finally:
        ix.close()
    assert not bad, "%s %s: %d cases differ from the oracle:\n%s" % (build, layout, len(bad), "\n".join(bad[:20]))


@pytest.mark.parametrize("build", T.BUILDS)
def test_grid_reaches_reductions_and_the_global_scratch(build, monkeypatch):
    """k_score's counting instantiation: at every -k from 2 to 32 some unit reduces over more than one rank round, and the
    batch has warps on the global scratch as well as warps in the shared pool; its records are the oracle's"""
    m = capi()
    set_env(monkeypatch, {"CFB_COUNT": "2"})
    ix = m.Index(T.index(build), 0)
    seen = []
    for k in (2, 3, 5, 8, 16, 17, 31, 32):
        for rs in ("se", "pe"):
            ctx = m.Context(ix, params(k, "default"))
            gn, grec = classify(ctx, T.batches()[rs])
            st = ctx.score_stats()
            ctx.close()
            assert_same(*oracle_records(build, rs, k, "default"), gn, grec)
            seen.append((k, rs, st["reduce_units"], st["reduce_rounds"], st["warps_global"], st["warps"]))
    ix.close()
    for k in (2, 3, 5, 8, 16, 17, 31, 32):
        assert any(s[0] == k and s[2] > 0 and s[3] > s[2] for s in seen), (build, k, seen)
    assert any(0 < s[4] < s[5] for s in seen), (build, seen)


# ------------------------------------------------------------------------------ centrifuge-class
@pytest.fixture(scope="module")
def read_files(tmp_path_factory):
    return T.write_reads(str(tmp_path_factory.mktemp("ties")))


def run_class(args, tmp, tag, env=None):
    tsv, rep, kr = str(tmp / (tag + ".tsv")), str(tmp / (tag + ".rep")), str(tmp / (tag + ".kreport"))
    p = subprocess.run([EXE] + list(args) + ["-S", tsv, "--report-file", rep, "--kreport-file", kr], stdout=subprocess.DEVNULL,
                       stderr=subprocess.PIPE, env=dict(os.environ, CFB_TEXT_STATS="1", **(env or {})))
    err = p.stderr.decode()
    assert p.returncode == 0, err
    t = re.search(r"text operator: (\d+) units in (\d+) spans .* (\d+) fallbacks\); record-level reader: (\d+) units", err)
    st = dict(text=int(t.group(1)), spans=int(t.group(2)), fallbacks=int(t.group(3)), host=int(t.group(4)))
    return tuple(open(x, "rb").read() for x in (tsv, rep)), open(kr, "rb").read(), st


def over_32(build, rs, k, case):
    return max(len(u) for u in units(*oracle_records(build, rs, k, case))) > 32


@pytest.mark.parametrize("inp", ["se_fq", "se_fa", "pe_fq"])
@pytest.mark.parametrize("build", T.BUILDS)
def test_cli_matches_reference(build, inp, read_files, tmp_path, monkeypatch):
    set_env(monkeypatch, {})
    base = T.index(build)
    rs = "pe" if inp.startswith("pe") else "se"
    n_units = T.batches()[rs].n
    bad, fell_back = [], 0
    for k in T.CLI_K:
        for case in T.CLI_CASES:
            args = read_files[inp][:1] + ["-x", base] + read_files[inp][1:] + ["-k", str(k)] + T.CLI_OPTIONS[case]
            want, want_k = reference_outputs(build, inp, k, case, args, tmp_path)
            got, kr, st = run_class(args, tmp_path, "text")
            got_h, kr_h, st_h = run_class(args + ["--host-parse"], tmp_path, "host")
            what = "k %d %s" % (k, case)
            if util.digest(got) != want or util.digest(kr) != want_k:
                bad.append("%s: text operator output differs from the reference's (%s)" % (what, st))
            if got_h != got or kr_h != kr:
                bad.append("%s: --host-parse writes other bytes" % what)
            if k > 32:
                ok = st["text"] == 0 and st["host"] == n_units
            elif over_32(build, rs, k, case):
                ok = st["fallbacks"] >= 1 and 0 < st["host"] <= n_units and st["text"] + st["host"] >= n_units
                fell_back += ok
            else:
                ok = st["fallbacks"] == 0 and st["host"] == 0 and st["text"] == n_units
            if not ok:
                bad.append("%s: reader statistics %s" % (what, st))
            if st_h["host"] != n_units:
                bad.append("%s: --host-parse statistics %s" % (what, st_h))
    assert not bad, "%s %s: %d cases:\n%s" % (build, inp, len(bad), "\n".join(bad))
    if build == "plain":
        assert fell_back > 0, "no unit of more than 32 records reached the text operator"


@pytest.mark.parametrize("case", ["default", "host"])
def test_cli_tie_sets_after_tie_free_spans(case, read_files, tmp_path, monkeypatch):
    """300 kB spans: the first two hold no tie sets, the third hundreds, and the outputs are the reference's.  That such a span
    needs the second copy of its tie sets is shown through the C ABI by test_tie_sets_beyond_the_speculative_copy."""
    set_env(monkeypatch, {})
    base = T.index("plain")
    args = read_files["mixed"][:1] + ["-x", base] + read_files["mixed"][1:] + ["-k", str(T.MIXED_K)] + T.CLI_OPTIONS[case]
    want, want_k = reference_outputs("plain", "mixed", T.MIXED_K, case, args, tmp_path)
    got, kr, st = run_class(args, tmp_path, "text", env={"CFB_TEXT_BLOCK": "300000"})
    util.assert_matches(got, want, case)
    util.assert_matches(kr, want_k, case)
    assert st["spans"] >= 3 and st["fallbacks"] == 0 and st["host"] == 0, st


# ------------------------------------------------------------------------------ per-taxon counters
def fold_rows(tsv):
    """numReads / numUniqueReads / singletons per taxid from the operator's rows: a read's first row counts as a read, as a
    unique read when it has one row, and as a singleton when that row also scores the read's maximum; later rows count as
    reads of their taxids"""
    out = {}
    lines = tsv.decode().rstrip("\n").split("\n")
    i = 0
    while i < len(lines):
        f = lines[i].split("\t")
        num, taxid, score, qlen = int(f[7]), int(f[2]), int(f[3]), int(f[6])
        best = (qlen - 15) ** 2 if qlen > 15 and f[1] != "unclassified" else 0
        c = out.setdefault(taxid, [0, 0, 0])
        c[0] += 1
        if num == 1:
            c[1] += 1
            c[2] += score >= best
        for j in range(1, num):
            out.setdefault(int(lines[i + j].split("\t")[2]), [0, 0, 0])[0] += 1
        i += num
    return out


def tie_sets_of_rows(tsv):
    """the tie sets the operator's rows imply: (num, its taxids in ascending order) of every read with more than one row whose
    first row scores the read's maximum, as a sorted list"""
    out = []
    lines = tsv.decode().rstrip("\n").split("\n")
    i = 0
    while i < len(lines):
        f = lines[i].split("\t")
        num, score, qlen = int(f[7]), int(f[3]), int(f[6])
        if num > 1 and score >= (qlen - 15) ** 2:
            out.append((num,) + tuple(sorted(int(lines[i + j].split("\t")[2]) for j in range(num))))
        i += num
    return sorted(out)


def tie_sets_of(r):
    """the tie sets text_wait returned: rows of stride k + 1, the count then the taxids"""
    return sorted(tuple(int(x) for x in row[:1 + int(row[0])]) for row in r["multi"])


@pytest.mark.parametrize("k", [2, 16, 32])
@pytest.mark.parametrize("build", T.BUILDS)
def test_text_species_counters_fold_the_rows(build, k, monkeypatch):
    """the operator's per-taxon counters and tie sets are those its own rows imply"""
    set_env(monkeypatch, {})
    m = capi()
    se = T.single_reads()
    text = b"".join(b">" + n.encode() + b"\n" + a.tobytes() + b"\n" for n, a in se)
    ix = m.Index(T.index(build), 0)
    wide = 0
    for case in ("default", "host", "genus"):
        ctx = m.Context(ix, params(k, case))
        ctx.text_submit(0, np.frombuffer(text, dtype=np.uint8).copy(), None, len(se), fasta=True)
        r = ctx.text_wait(0)
        assert not r["irregular"] or (case == "host" and over_32(build, "se", k, case)), (k, case)
        if not r["irregular"]:
            sp = ctx.text_species()
            got = {int(t): [int(a), int(b), int(c)] for t, a, b, c in zip(sp["taxid"], sp["n_reads"], sp["n_unique"], sp["n_obs1"]) if a or b or c}
            assert got == fold_rows(r["tsv"]), (build, k, case)
            assert r["multi"].shape[1] == k + 1, r["multi"].shape
            want = tie_sets_of_rows(r["tsv"])
            assert tie_sets_of(r) == want, (build, k, case)
            wide += any(t[0] > 16 for t in want)
        ctx.close()
    ix.close()
    assert k < 32 or wide, "no tie set of more than 16 taxa"


def test_tie_sets_beyond_the_speculative_copy(monkeypatch):
    """cfb_text_wait copies ahead as many tie sets as earlier spans suggest (cfb_text_submit: n x multi_ratio x 1.2 + 256,
    multi_ratio starting at 0.05 and decaying by 0.98 a span) and fetches the rest once it knows their number.  Two tie-free
    spans, then a span with several hundred tie sets of up to 32 taxa: more than the speculative copy holds, and all of them
    the ones its rows imply."""
    set_env(monkeypatch, {})
    m = capi()
    free, heavy = T.mixed_reads()
    half = len(free) // 2
    ix = m.Index(T.index("plain"), 0)
    ctx = m.Context(ix, params(T.MIXED_K, "default"))
    ratio = 0.05
    for reads in (free[:half], free[half:], heavy):
        text = b"".join(b">" + n.encode() + b"\n" + a.tobytes() + b"\n" for n, a in reads)
        ctx.text_submit(0, np.frombuffer(text, dtype=np.uint8).copy(), None, len(reads), fasta=True)
        r = ctx.text_wait(0)
        assert not r["irregular"]
        spec = min(len(reads), int(len(reads) * ratio * 1.2) + 256)
        assert tie_sets_of(r) == tie_sets_of_rows(r["tsv"])
        ratio = max(ratio * 0.98, r["n_multi"] / len(reads))
    ctx.close(); ix.close()
    assert r["n_multi"] > spec and max(t[0] for t in tie_sets_of(r)) == 32, (r["n_multi"], spec)


def fold_records(b, n, rec, k):
    """the record-level counters' contract: a unit counts its records of the best score, the first k of them in record order;
    a unit without records counts as taxid 0"""
    out = {}
    for u, rs in enumerate(units(n, rec)):
        if len(rs) == 0:
            c = out.setdefault(0, [0, 0, 0]); c[0] += 1; c[1] += 1; c[2] += 1
            continue
        best = int(rs["score"].max())
        top = [int(r["taxid"]) for r in rs if int(r["score"]) == best][:k]
        L = [int(b.len1[u])] + ([int(b.len2[u])] if b.paired else [])
        mx = sum((x - 15) ** 2 for m, x in enumerate(L) if (b.flags[u] >> m) & 1 and x > 15)
        c = out.setdefault(top[0], [0, 0, 0]); c[0] += 1
        if len(top) == 1:
            c[1] += 1; c[2] += best >= mx
        for t in top[1:]:
            out.setdefault(t, [0, 0, 0])[0] += 1
    return out


@pytest.mark.parametrize("build", T.BUILDS)
def test_record_level_counters_follow_the_hit_map_order(build, monkeypatch):
    """with more than k tied best records (the host set) the counters take the first k in record order"""
    set_env(monkeypatch, {})
    m = capi()
    ix = m.Index(T.index(build), 0)
    wide = 0
    for rs in ("se", "pe"):
        b = T.batches()[rs]
        for k, case in ((1, "default"), (5, "default"), (16, "genus"), (2, "host"), (16, "host"), (32, "host"), (40, "host")):
            ctx = m.Context(ix, params(k, case))
            ctx.count_records(True)
            gn, grec = classify(ctx, b)
            tax = ctx.counts_taxids()
            cnt = ctx.counts_dense()
            ctx.close()
            assert_same(*oracle_records(build, rs, k, case), gn, grec)
            got = {int(t): [int(x) for x in cnt[:, i]] for i, t in enumerate(tax) if cnt[:, i].any()}
            assert got == fold_records(b, gn, grec, k), (build, rs, k, case)
            wide += any(len(u) > k for u in units(gn, grec))
    ix.close()
    assert wide, "no unit has more tied best records than -k"
