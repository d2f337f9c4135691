"""Abundance EM on the device (SURVEY.md 8f rank 3): `cfb_em_abundance` must produce the very doubles of the
reference's sequential loops (aln_sink.h:196-495).  The checkers here are a plain-Python restatement of those loops
(Python floats are IEEE doubles and the loops add in the same order), its order-exact numpy form for the large tables,
the product's host loop, and the reference binary's reports and EM lines through the CLI."""
import lzma
import os

import numpy as np
import pytest

import util
from util_em import (ADV_CASES, BENCH, LARGE, MATRIX, adv_reference_em_lines, bits, device_em, em_numpy, em_python, host_em,
                     problem, random_problem, run_class)

pytestmark = pytest.mark.gpu

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")


@pytest.mark.parametrize("seed,n,K", [(1, 7, 30), (2, 60, 400), (3, 300, 3000), (4, 5, 3)])
def test_device_em_is_bit_identical_to_the_sequential_loops(seed, n, K):
    count, key_off, target, length, p0 = random_problem(seed, n, K)
    want, want_it, want_diff = em_python(count, key_off, target, length, list(p0))
    got, it, diff = device_em(count, key_off, target, length, p0)
    assert it == want_it
    assert np.array_equal(bits(got), bits(want))
    assert diff == want_diff


@pytest.mark.parametrize("seed,n,K,kind", MATRIX + [LARGE, BENCH])
def test_device_em_matches_numpy_restatement_and_host_loop(seed, n, K, kind):
    """Device == em_numpy == host loop in the bits of p (NaN signs included), the iteration count and the bits of the
    last difference: block and 8-wide tail edges, empty / zero-psum / duplicate / 500-target keys, a species in 40 % of
    the keys, counts and sizes that are not exact doubles, fixed points, 100+ iterations, NaN up to the cap, and the
    tables above the 2^18 contributions that select the device in centrifuge-class."""
    pr = problem(seed, n, K, kind)
    want, want_it, want_diff = em_numpy(*pr)
    for got, it, diff in (device_em(*pr), host_em(*pr)):
        assert (it, bits([diff])[0]) == (want_it, bits([want_diff])[0])
        assert np.array_equal(bits(got), bits(want))
    if kind == "nan":
        assert want_it == 10000 and np.all(bits(want) == np.uint64(0xFFF8000000000000))   # x86's NaN: the report prints -nan


def adv_reads_file(tmp_path):
    reads = str(tmp_path / "reads.fa")
    with lzma.open(os.path.join(util.GOLDEN, "adv.reads.fa.xz")) as f, open(reads, "wb") as g:
        g.write(f.read())
    return reads


@pytest.mark.parametrize("case,opts", [("default", []), ("k50", ["-k", "50"]), ("family", ["--classification-rank", "family"])])
def test_cli_report_with_device_em_matches_reference_golden(case, opts, tmp_path):
    assert opts == ADV_CASES[case]
    base = util.golden_index("adv")
    reads = adv_reads_file(tmp_path)
    outs = {}
    for mode in ("1", "0"):
        rep, lines, _ = run_class(EXE, ["-f", "-x", base, "-U", reads] + opts, tmp_path, env=dict(os.environ, CFB_GPU_EM=mode))
        outs[mode] = (rep, lines)
        with open(os.path.join(util.GOLDEN, "adv.%s.report.tsv" % case), "rb") as f:
            assert rep == f.read()
        util.assert_matches(lines, adv_reference_em_lines(case, base, reads, tmp_path), case, "CFB_GPU_EM=" + mode)
    assert outs["1"] == outs["0"]          # same iteration count and final difference as the host loop


# A workload whose tie-set table crosses the 2^18 contributions at which centrifuge-class moves the EM to the device by
# itself: 10 genera of 30 near-identical species (0.5 % divergence), 60 000 exact 100-base reads, -k 50.  Reads tie
# among the species that carry no mutation under them, so nearly every read is a distinct key of ~18 species:
# 300 species, 18 416 keys, 334 352 contributions (counted from the reference's TSV through flatten()).
LARGE_INDEX = ("em_large", 10, 30, 20000, 5)


def large_workload(tmp):
    base = util.build_index(*LARGE_INDEX, div=0.005)
    seqs = util.synth.make_genomes(*LARGE_INDEX[1:], div=0.005)
    reads = os.path.join(str(tmp), "large.fa")
    util.synth.write_fasta(reads, util.synth.sample_reads(seqs, 60000, 100, seed=71, sub=0.0, nrate=0.0, random_frac=0.0))
    return ["-f", "-x", base, "-U", reads, "-k", "50"]


def large_reference(args, tmp):
    return util.reference("em/large_table", lambda: run_class(util.REF_CLASS, args, tmp)[:2])


def em_diag(stderr):
    ln = [x for x in stderr.splitlines() if x.startswith("[cfb] abundance EM: ")]
    assert len(ln) == 1, stderr[-2000:]
    w = ln[0].split()
    return int(w[3]), int(w[5]), int(w[7]), w[-1]


def test_cli_large_table_runs_the_em_on_the_device_by_itself(tmp_path):
    args = large_workload(tmp_path)
    env = {k: v for k, v in os.environ.items() if k != "CFB_GPU_EM"}
    rep, lines, err = run_class(EXE, args, tmp_path, env=dict(env, CFB_TEXT_STATS="1"))
    n, K, T, where = em_diag(err)
    assert where == "device" and T >= 1 << 18, (n, K, T, where)
    util.assert_matches((rep, lines), large_reference(args, tmp_path), (n, K, T))
    rep0, lines0, err0 = run_class(EXE, args, tmp_path, env=dict(env, CFB_TEXT_STATS="1", CFB_GPU_EM="0"))
    assert em_diag(err0) == (n, K, T, "host")
    assert (rep0, lines0) == (rep, lines)


# NaN: a --size-table that gives one leaf the genome size 0 turns the start vector into inf / inf, every value into NaN,
# and the loop runs to its cap; x86's NaN is negative, so the reference's report prints -nan.
NAN_INDEX = (3, 4, 20000, 9)


def nan_index(tmp):
    """The index with a size table, built by the project's builder; its files must be the reference builder's."""
    from centrifuge_b200 import capi
    d = str(tmp)
    util.synth.write_genomes(d, *NAN_INDEX)
    with open(d + "/sizes.tsv", "w") as f:
        f.write("1001\t5000000\n1002\t0\n")
    tax = dict(conversion_table=d + "/conv.tsv", taxonomy_tree=d + "/nodes.dmp", name_table=d + "/names.dmp")

    def ref():
        import subprocess
        subprocess.check_call([util.REF_BUILD, "-p", "4", "--conversion-table", tax["conversion_table"], "--taxonomy-tree", tax["taxonomy_tree"],
                               "--name-table", tax["name_table"], "--size-table", d + "/sizes.tsv", d + "/genomes.fa", d + "/ref"],
                              stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        return [open("%s/ref.%s.cf" % (d, k), "rb").read() for k in "1234"]
    want = util.reference("build/size_table_zero", ref)
    if util.RECORD:
        return d + "/ref"
    capi.build_index(capi.build_opts(d + "/mine", fasta=[d + "/genomes.fa"], size_table=d + "/sizes.tsv", **tax))
    util.assert_matches([open("%s/mine.%s.cf" % (d, k), "rb").read() for k in "1234"], want, "size table")
    return d + "/mine"


def nan_workload(tmp):
    base = nan_index(tmp)
    seqs = util.synth.make_genomes(*NAN_INDEX)
    reads = os.path.join(str(tmp), "nan.fa")
    util.synth.write_fasta(reads, util.synth.sample_reads(seqs, 3000, 100, seed=72, sub=0.0, nrate=0.0))
    return ["-f", "-x", base, "-U", reads]


def nan_reference(args, tmp):
    return util.reference("em/size_zero", lambda: run_class(util.REF_CLASS, args, tmp)[:2])


def test_cli_size_table_zero_prints_the_reference_nan(tmp_path):
    args = nan_workload(tmp_path)
    want = nan_reference(args, tmp_path)
    for mode in ("1", "0"):
        rep, lines, _ = run_class(EXE, args, tmp_path, env=dict(os.environ, CFB_GPU_EM=mode))
        assert b"\t-nan\n" in rep and lines[0].endswith(": 10000") and lines[1].endswith(": -nan"), (rep, lines)
        util.assert_matches((rep, lines), want, "CFB_GPU_EM=" + mode)
