"""Abundance EM, host form (`cfb_em_abundance_host`, the loop `centrifuge-class` runs for small tie-set tables): the very
doubles and iteration count of the reference's sequential loops, checked against a plain-Python restatement, its
order-exact numpy form, and through both against the reference binary's reports and EM lines."""
import lzma
import os

import numpy as np
import pytest

import util
from util_em import (ADV_CASES, LARGE, MATRIX, adv_reference_em_lines, bits, em_numpy, em_python, em_stderr_lines, flatten,
                     fmt_double, host_em, index_tree, observed_from_tsv, problem, random_problem, report_abundance)


@pytest.mark.parametrize("seed,n,K", [(1, 7, 30), (2, 60, 400), (3, 300, 3000), (4, 5, 3), (5, 40, 1)])
def test_host_em_is_bit_identical_to_the_sequential_loops(seed, n, K):
    count, key_off, target, length, p0 = random_problem(seed, n, K)
    want, want_it, want_diff = em_python(count, key_off, target, length, list(p0))
    got, it, diff = host_em(count, key_off, target, length, p0)
    assert it == want_it
    assert np.array_equal(bits(got), bits(want))
    assert diff == want_diff


@pytest.mark.parametrize("seed,n,K,kind", [m for m in MATRIX if m[3] != "nan"])
def test_numpy_restatement_is_bit_identical_to_the_loops(seed, n, K, kind):
    """em_numpy (the checker of the large tables) == em_python in every bit, iteration count and last difference."""
    count, key_off, target, length, p0 = problem(seed, n, K, kind)
    want, want_it, want_diff = em_python(count, key_off, target, length, list(p0))
    got, it, diff = em_numpy(count, key_off, target, length, p0)
    assert (it, bits([diff])[0]) == (want_it, bits([want_diff])[0])
    assert np.array_equal(bits(got), bits(want))


@pytest.mark.parametrize("seed,n,K,kind", MATRIX + [LARGE])
def test_host_em_matches_numpy_restatement(seed, n, K, kind):
    """The product's host loop == em_numpy on every shape, the iteration cap and NaN (bit patterns, sign included) too."""
    pr = problem(seed, n, K, kind)
    want, want_it, want_diff = em_numpy(*pr)
    got, it, diff = host_em(*pr)
    assert (it, bits([diff])[0]) == (want_it, bits([want_diff])[0])
    assert np.array_equal(bits(got), bits(want))
    if kind == "slow":
        assert it >= 100
    if kind == "singletons":
        assert it == 1                                   # a fixed point after one step: ssv == 0 at iteration 1
    if n == 1:
        assert it == 0 and diff == 0.0                   # ssv == 0 at iteration 0
    if kind == "underflow":
        assert it == 0 and 0.0 < diff < 1e-150           # ssv == 0 while p still moves: the third step must stay off
    if kind == "nan":
        assert it == 10000 and np.isnan(diff) and np.all(bits(got) == np.uint64(0xFFF8000000000000))
    if kind == "skew":
        assert sum(0 in pr[2][pr[1][k]:pr[1][k + 1]] for k in range(K)) >= K // 4
    if kind == "wide":
        assert max(np.diff(pr[1])) >= 500


def test_large_table_is_order_sensitive():
    """A reordered sum over species (np.sum adds pairwise) changes the result of the large table: the bit-exact checks
    above would catch a kernel that adds in another order."""
    pr = problem(*LARGE)
    assert pr[1][-1] >= 1 << 18
    a = em_numpy(*pr)
    b = em_numpy(*pr, species_sum=np.sum)
    assert not (np.array_equal(bits(a[0]), bits(b[0])) and a[2] == b[2])


@pytest.mark.parametrize("case", sorted(ADV_CASES))
def test_restatement_reproduces_reference_report_and_em_lines(case, adv_base, adv_reads, tmp_path):
    """Golden classification TSV -> observed_from_tsv -> flatten -> em_numpy gives the golden report's abundance column
    and the reference binary's iteration count and last difference: the restatement is pinned to the reference itself."""
    with lzma.open(os.path.join(util.GOLDEN, "adv.%s.tsv.xz" % case)) as f:
        rows = f.read().decode().splitlines()[1:]
    with open(os.path.join(util.GOLDEN, "adv.%s.report.tsv" % case), "rb") as f:
        rep = report_abundance(f.read())
    observed = observed_from_tsv(rows)
    count, key_off, target, length, p0, taxids = flatten(observed, index_tree(adv_base), {t: s for t, (s, _) in rep.items()})
    p, it, diff = em_numpy(count, key_off, target, length, p0)
    assert [fmt_double(x) for x in p] == [rep[t][1] for t in taxids]
    assert all(rep[t][1] == "0.0" for t in rep if t not in taxids)
    util.assert_matches(em_stderr_lines(it, diff), adv_reference_em_lines(case, adv_base, adv_reads, tmp_path), case)
    if not taxids:
        assert case == "family" and it == 0              # every tie at family rank: no leaf, nothing to iterate
        return
    # and the product's host loop on the same table
    got, it2, diff2 = host_em(count, key_off, target, length, p0)
    assert (it2, diff2) == (it, diff) and np.array_equal(bits(got), bits(p))
