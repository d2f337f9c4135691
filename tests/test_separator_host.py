"""`centrifuge-class --separator` on the CPU: option handling, and the per-input sequence of rows, separator lines and
reports of the record-level path.  The cfb_test_separator hook runs that path around classification records from the
oracle and must reproduce the bytes the unmodified reference binary writes for the same inputs (recorded digests)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import util
import util_separator as us
from test_host_path import dump_reads

EXE = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")
CASES = {"default": [], "k1": ["-k", "1"], "k50": ["-k", "50"], "no_abundance": ["--no-abundance"]}


def test_arg_desc_lists_separator():
    out = subprocess.run([EXE, "--arg-desc"], stdout=subprocess.PIPE, check=True).stdout
    assert b"separator\t0" in out.split(b"\n")


def test_kreport_file_with_separator_is_refused(adv_base, adv_reads, tmp_path):
    p = subprocess.run([EXE, "-f", "-x", adv_base, "-U", adv_reads, "--separator", "--kreport-file", "k.txt", "-S", "o.tsv"],
                       cwd=str(tmp_path), stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
    assert p.returncode == 1 and b"--kreport-file" in p.stderr and b"--separator" in p.stderr, p.stderr
    assert os.listdir(str(tmp_path)) == []


def oracle_records(lib, oracle, files, k, tmp):
    """per input: (units, records per unit, records) from the oracle, for the reads the product's reader reads"""
    out = []
    for a, b in files:
        m1 = dump_reads(lib, a, False, (0, 0), tmp)
        bt = util.Batch(m1, dump_reads(lib, b, False, (0, 0), tmp)) if b else util.Batch(m1)
        if bt.n == 0:
            out.append((0, np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=util.REC)))
            continue
        on, orec, _ = oracle.classify(bt, util.make_oparams(k=k))
        out.append((bt.n, on, orec))
    return out


def hook_run(lib, base, files, recs, k, abundance, cwd, capfd):
    """cfb_test_separator over the inputs in cwd: (TSV, reports, stderr lines), as util_separator.run returns them"""
    os.makedirs(str(cwd))
    n = len(files)
    rec_off = np.concatenate([[0], np.cumsum(np.concatenate([r[1] for r in recs]))]).astype(np.uint32)
    allrecs = np.ascontiguousarray(np.concatenate([r[2] for r in recs]))
    units = (C.c_uint64 * n)(*[r[0] for r in recs])
    pa = (C.c_char_p * n)(*[a.encode() for a, _ in files])
    pb = (C.c_char_p * n)(*[b.encode() if b else None for _, b in files])
    out = os.path.join(str(cwd), "out.tsv")
    here = os.getcwd()
    capfd.readouterr()
    os.chdir(str(cwd))
    try:
        rc = lib.cfb_test_separator(base.encode(), C.c_int(n), pa, pb, C.c_int(0), C.c_int(k), C.c_int(1 if abundance else 0), units,
                                    rec_off.ctypes.data_as(C.POINTER(C.c_uint32)), allrecs.ctypes.data_as(C.c_void_p), out.encode())
    finally:
        os.chdir(here)
    err = capfd.readouterr().err
    assert rc == 0, (rc, err)
    return open(out, "rb").read(), us.reports(cwd), us.stderr_lines(err.encode())


@pytest.mark.parametrize("case", sorted(CASES))
def test_per_input_reports_match_reference(case, adv_base, adv_reads, tmp_path, capfd):
    util.ensure_oracle()
    lib = C.CDLL(util.PRODUCT_LIB)
    files, args = us.write_inputs(tmp_path, us.adv_regular_reads(adv_reads))
    k = int(CASES[case][1]) if case.startswith("k") else 5
    abundance = case != "no_abundance"
    o = util.Oracle(adv_base)
    recs = oracle_records(lib, o, files, k, tmp_path)
    o.close()
    got = hook_run(lib, adv_base, files, recs, k, abundance, tmp_path / "hook", capfd)
    want, _ = us.reference_outputs(case, ["-q", "-x", adv_base] + args + CASES[case], tmp_path)
    util.assert_matches(got, want, case)
    assert got[0].count(us.SEP) == len(files) and len(got[1]) == len(files)
    assert got[1][3][1].count(b"\n") == 1                           # the empty input: header only
    if case == "k50":
        # the reference keeps the tie sets of earlier inputs: the last input's report, alone, has the same counts but
        # another abundance column
        alone = hook_run(lib, adv_base, files[-1:], recs[-1:], k, abundance, tmp_path / "alone", capfd)[1][0][1]
        carried = got[1][-1][1]
        def cols(rep, sl):
            return [tuple(ln.split(b"\t")[sl]) for ln in rep.split(b"\n")]
        assert cols(alone, slice(0, 6)) == cols(carried, slice(0, 6))
        assert cols(alone, slice(6, 7)) != cols(carried, slice(6, 7))
