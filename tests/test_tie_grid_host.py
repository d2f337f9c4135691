"""CPU: the oracle and the host-compiled product logic on the tie-rich fixture (util_ties.py) across -k 1 to 64, before the device
is compared with them.

- The oracle's file driver writes the reference binary's TSV and report (recorded digests) for single-end FASTQ and FASTA and
  paired FASTQ, on both builds, at every -k of util_ties.CLI_K with the default options, the host set and --classification-rank
  genus; cfb_kreport on those rows writes what the reference's centrifuge-kreport writes.
- cf_logic.h compiled for the host (util.HostLogic) gives the oracle's records, unit by unit, over the whole -k / option grid.
- The fixture reaches what it is for: every tie group size, a unit with more than 32 tied host records, and every repeat's
  records moving between the two -k values around its ihits threshold."""
import concurrent.futures
import ctypes as C
import functools
import os

import numpy as np
import pytest

import util
import util_ties as T


@functools.lru_cache(None)
def oracle_records(build, rs, k, case):
    o = util.Oracle(T.index(build))
    n, rec, _ = o.classify(T.batches()[rs], util.make_oparams(k=k, **T.OPTIONS[case]))
    o.close()
    return n, rec


def units(n, rec):
    off = np.concatenate([[0], np.cumsum(n.astype(np.int64))])
    return [rec[off[i]:off[i + 1]] for i in range(len(n))]


def se_index(prefix):
    return [i for i, (nm, _) in enumerate(T.single_reads()) if nm.startswith(prefix)]


@pytest.mark.parametrize("build", T.BUILDS)
def test_every_tie_group_size_is_reached(build):
    """a read of each genus block ties among exactly S sequences at a -k >= S; so do the family block's 54"""
    for g, S in enumerate(T.SPECIES):
        us = units(*oracle_records(build, "se", 64, "default"))
        got = [len(us[i]) for i in se_index("g%d_" % g)]
        assert S in got, (build, g, S, got)
        assert all(len(set(u["score"])) == 1 for u in (us[i] for i in se_index("g%d_" % g)) if len(u) == S)
    us = units(*oracle_records(build, "se", 64, "default"))
    assert 54 in [len(us[i]) for i in se_index("f10_")]


def test_host_set_gives_units_over_32_records():
    """--host-taxids keeps every tied host record: the 40-sequence genus gives units of 40 records of one score at -k <= 32"""
    for build, k in (("plain", 1), ("plain", 16), ("plain", 32), ("cid", 16)):
        us = units(*oracle_records(build, "se", k, "host"))
        assert any(len(u) > 32 and len(set(u["score"])) == 1 for u in us), (build, k)


@pytest.mark.parametrize("build", T.BUILDS)
def test_repeats_move_at_their_ihits_threshold(build):
    """a repeat of c copies is dropped at every -k whose ihits is below c: its reads' records differ between the two -k values
    of the grid around the threshold"""
    moved = set()
    for i, c in enumerate(T.COPIES):
        idx = se_index("rep%d_" % c)
        for k0, k1 in zip(T.K_GRID, T.K_GRID[1:]):
            if T.ihits(build, k0) < c <= T.ihits(build, k1):
                a = units(*oracle_records(build, "se", k0, "default"))
                b = units(*oracle_records(build, "se", k1, "default"))
                assert all(len(a[j]) == 0 and len(b[j]) > 0 for j in idx), (build, c, k0, k1)
                moved.add(c)
    want = {21, 33, 65, 129} if build == "cid" else {201, 241}
    assert want <= moved, (build, moved)


@pytest.mark.parametrize("rs", ["se", "pe"])
@pytest.mark.parametrize("build", T.BUILDS)
def test_host_logic_matches_oracle_over_the_grid(build, rs):
    h = util.HostLogic(T.index(build))
    keys = [(k, case) for k in T.K_GRID for case in T.OPTIONS]
    with concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        list(ex.map(lambda a: oracle_records(build, rs, *a), keys))
    bad = []
    for k, case in keys:
        hn, hrec, _ = h.classify(T.batches()[rs], util.make_oparams(k=k, **T.OPTIONS[case]))
        on, orec = oracle_records(build, rs, k, case)
        if not (np.array_equal(on, hn) and np.array_equal(orec, hrec)):
            d = np.nonzero(on != hn)[0]
            bad.append("k %d %s: %d units differ in count (first %s)" % (k, case, len(d), d[:5]) if len(d) else "k %d %s: records differ" % (k, case))
    h.close()
    assert not bad, "%s %s: %d cases differ from the oracle:\n%s" % (build, rs, len(bad), "\n".join(bad[:20]))


# ------------------------------------------------------------------------------ the oracle's file driver and the Kraken-style report
def kreport_of_tsv(base, tsv, out):
    lib = C.CDLL(util.PRODUCT_LIB)
    rc = lib.cfb_kreport(base.encode(), tsv.encode(), out.encode(), C.c_int(0), C.c_int(0), C.c_longlong(0), C.c_int(0), C.c_longlong(0))
    assert rc == 0
    with open(out, "rb") as f:
        return f.read()


def ref_kreport(base, tsv, tmp):
    import subprocess
    p = subprocess.run(["perl", util.ref_script("centrifuge-kreport", tmp), "-x", base, tsv], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    assert p.returncode == 0
    return p.stdout


def reference_outputs(build, inp, k, case, args, tmp):
    """recorded digests of the reference's (TSV, report) and of centrifuge-kreport on that TSV"""
    key = T.cli_key(build, inp, k, case)
    tsv, rep = str(tmp / "ref.tsv"), str(tmp / "ref.rep")
    run = lambda: util.run_cli(util.REF_CLASS, args, tsv, rep)           # noqa: E731
    want = util.reference(key, run)
    want_k = util.reference(key + "/kreport", lambda: ref_kreport(args[args.index("-x") + 1], tsv, tmp))
    return want, want_k


@pytest.mark.parametrize("inp", ["se_fq", "se_fa", "pe_fq"])
@pytest.mark.parametrize("build", T.BUILDS)
def test_oracle_file_driver_matches_reference(build, inp, tmp_path):
    util.ensure_oracle()
    base = T.index(build)
    files = T.write_reads(str(tmp_path / "reads"))
    bad = []
    for k in T.CLI_K:
        for case in T.CLI_CASES:
            args = files[inp][:1] + ["-x", base] + files[inp][1:] + ["-k", str(k)] + T.CLI_OPTIONS[case]
            want, want_k = reference_outputs(build, inp, k, case, args, tmp_path)
            tsv = str(tmp_path / "o.tsv")
            got = util.run_cli(util.ORACLE_BIN, args, tsv, str(tmp_path / "o.rep"))
            if util.digest(got) != want:
                bad.append("k %d %s: TSV / report" % (k, case))
            if util.digest(kreport_of_tsv(base, tsv, str(tmp_path / "k.txt"))) != want_k:
                bad.append("k %d %s: kreport" % (k, case))
    assert not bad, "%s %s: %d cases differ from the reference:\n%s" % (build, inp, len(bad), "\n".join(bad))


@pytest.mark.parametrize("case", ["default", "host"])
def test_oracle_file_driver_matches_reference_on_the_mixed_file(case, tmp_path):
    """tie-free reads first, tie-heavy reads after them (the file the device's tie-set copy is tested on)"""
    util.ensure_oracle()
    base = T.index("plain")
    files = T.write_reads(str(tmp_path / "reads"))
    args = files["mixed"][:1] + ["-x", base] + files["mixed"][1:] + ["-k", str(T.MIXED_K)] + T.CLI_OPTIONS[case]
    want, want_k = reference_outputs("plain", "mixed", T.MIXED_K, case, args, tmp_path)
    tsv = str(tmp_path / "o.tsv")
    util.assert_matches(util.run_cli(util.ORACLE_BIN, args, tsv, str(tmp_path / "o.rep")), want, case)
    util.assert_matches(kreport_of_tsv(base, tsv, str(tmp_path / "k.txt")), want_k, case)
