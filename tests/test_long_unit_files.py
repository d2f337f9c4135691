"""The oracle's file driver (cf_oracle) on the long-unit read files of util_long.py writes the reference binary's TSV and report:
repeat-rich reads over 60 000 bases, long twins, long mates that fail the N filter, and reads of 59 999 - 60 010 bases trimmed
across the threshold.  The device tests of test_gpu_long_unit_grid.py take the oracle as their reference on these reads."""
import pytest

import util
import util_long as L


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("longunits"))
    return {c[0]: c for c in L.cli_cases(d, util.golden_index("adv"))}


def test_cases_cross_the_threshold():
    """the threshold file holds reads of 59 999, 60 000, 60 001 and 60 010 bases; the trims move units to both paths"""
    got = {c[0]: c[3] for c in L.cli_cases()}
    assert [n for n, a in L.cli_read_files()["th"] if n.startswith("t")] == ["t%d" % n for n in L.THRESH]
    assert got["th_0_0"] == 2 and got["th_0_1"] == 1 and got["th_1_0"] == 1 and got["th_10_0"] == 0 and got["th_0_2"] == 1
    assert got["se_fq"] == 6 and got["pe_fq"] == 6


@pytest.mark.parametrize("case", [c[0] for c in L.cli_cases()])
def test_oracle_file_driver_matches_reference(cases, case, tmp_path):
    util.ensure_oracle()
    key, args, _, _ = cases[case]
    want = L.ref_digest(key, args, tmp_path)
    got = util.run_cli(util.ORACLE_BIN, args, str(tmp_path / "o.tsv"), str(tmp_path / "o.rep"))
    util.assert_matches(got, want, case)
