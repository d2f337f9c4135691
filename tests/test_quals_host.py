"""Quality encodings without a GPU: the shared conversions (cf_quals.h) against a Python restatement over every byte and
every integer from -20 to 300 in every mode; the record-level reader (cfb_test_parse_quals) against the reference
binary's readID / readQual rows, one per read, for every option and its combinations, trims and integer quirks; the
reference's refusals; and the option table."""
import ctypes as C
import os
import subprocess

import pytest

import util
import util_quals as U

CLI = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(util.ROOT, "tests", "native", "quals_host.cpp")
    hdr = os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_quals.h")
    out = os.path.join(util.CACHE, "libquals_host.so")
    os.makedirs(util.CACHE, exist_ok=True)
    if not os.path.exists(out) or max(os.path.getmtime(src), os.path.getmtime(hdr)) > os.path.getmtime(out):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out + ".tmp", src])
        os.replace(out + ".tmp", out)
    lib = C.CDLL(out)
    lib.q_steps.restype = C.c_uint32
    return lib


def test_solexa_table_is_the_formula(shim):
    """the steps mask is complete (non-zero) and every Solexa value from -20 to 300 converts as the formula does"""
    assert shim.q_steps() != 0
    got = (C.c_int * 321)()
    shim.q_ints(1, -20, 300, got)
    assert [got[i] - 33 for i in range(321)] == [U.solexa_to_phred(q) for q in range(-20, 301)]
    # the conversion the reference's table holds at its edges
    assert [U.solexa_to_phred(q) for q in (-11, -10, -9, 0, 9, 10, 255)] == [0, 0, 1, 3, 10, 10, 255]


@pytest.mark.parametrize("solexa,phred64", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_character_conversion(shim, solexa, phred64):
    got = (C.c_int * 256)()
    shim.q_chars(solexa, phred64, got)
    for b in range(256):
        want = U.char_to_phred33(b, solexa, phred64)
        assert got[b] == (-1 if want is None else want), (b, solexa, phred64)


@pytest.mark.parametrize("solexa", [0, 1])
def test_integer_conversion(shim, solexa):
    got = (C.c_int * 321)()
    shim.q_ints(solexa, -20, 300, got)
    for i, v in enumerate(range(-20, 301)):
        assert got[i] == U.int_to_phred33(v, solexa), v
    if not solexa:
        assert all(got[i] < 33 for i in range(20)) and got[20] == 33       # negatives are refused, 0 is '!'


def test_atoi(shim):
    for s, v in (("", 0), ("12", 12), ("\t7", 7), ("+5", 5), ("-3", -3), ("12x9", 12), ("x1", 0), ("0003", 3), ("-", 0),
                 ("99999999999", 2 ** 31 - 1), ("-99999999999", -2 ** 31)):
        assert shim.q_atoi(s.encode()) == v, s


def test_options_apply_in_order(shim):
    for opt, bits in (("phred64", 2), ("phred64-quals", 2), ("solexa1.3-quals", 2), ("solexa-quals", 1), ("int-quals", 4), ("integer-quals", 4)):
        assert shim.q_apply(0, opt.encode()) == bits
    assert shim.q_apply(7, b"phred33") == 4 and shim.q_apply(7, b"phred33-quals") == 4       # integer stays
    assert shim.q_apply(0, b"phred32") == -1


# ----------------------------------------------------------------------------- the reader against the binary
READER_CASES = [(m, "se") for m in U.MODES] + [(m, w) for m in U.MAIN for w in ("trim", "long")] + \
               [(m, w) for m in U.MAIN if U.is_int(m) for w in ("quirks", "line4096")]


def _read_id(name):
    if len(name) >= 2 and name[-2:] in (b"/1", b"/2", b"/3"):
        name = name[:-2]
    for i, c in enumerate(name):
        if chr(c).isspace():
            return name[:i]
    return name


def product_reader(path, mode, trims, out, capfd):
    """(failed, error lines, `readID\\treadQual` rows) of the record-level reader under the mode's options"""
    lib = C.CDLL(util.PRODUCT_LIB)
    capfd.readouterr()
    rc = lib.cfb_test_parse_quals(path.encode(), C.c_int(0), C.c_int(trims[0]), C.c_int(trims[1]), C.c_uint32(0), None,
                                  U.opt_names(mode).encode(), out.encode())
    err = capfd.readouterr().err.encode()
    if rc != 0:
        assert rc == 1
        return True, U.error_lines(err), b""
    rows = [b"readID\treadQual\n"]
    with open(out, "rb") as f:
        for line in f.read().split(b"\n")[:-1]:
            name, _, _, _, q = line.split(b"\t")
            rows.append(_read_id(name) + b"\t" + bytes.fromhex(q.decode()) + b"\n")
    return False, [], b"".join(rows)


@pytest.mark.parametrize("mode,which", READER_CASES, ids=["%s-%s" % c for c in READER_CASES])
def test_reader_matches_reference(adv_base, tmp_path, capfd, mode, which):
    args = U.inputs(os.path.join(util.CACHE, "quals_inputs"), mode)[which]
    trims = (3, 2) if which == "trim" else (0, 0)
    opts = U.MODES[mode][0] + ["-k", "1", "--tab-fmt-cols", "readID,readQual"]
    want = U.reference("reader/%s/%s" % (which, mode), lambda: U.run_ref_error(util.REF_CLASS, adv_base, opts + args, tmp_path))
    if util.RECORD:
        return
    got = product_reader(args[-1], mode, trims, str(tmp_path / "dump.txt"), capfd)
    util.assert_matches(got, want, mode, which)


@pytest.mark.parametrize("case", sorted(U.ERRORS))
def test_refusals_match_reference(adv_base, tmp_path, capfd, case):
    mode, trims = U.ERRORS[case]
    path = U.write(os.path.join(str(tmp_path), "bad.fq"), U.fastq(U.error_records(case)))
    targs = ["-5", str(trims[0]), "-3", str(trims[1])]
    want = U.reference("error/" + case, lambda: U.run_ref_error(util.REF_CLASS, adv_base, U.MODES[mode][0] + targs + ["-U", path], tmp_path))
    if util.RECORD:
        return
    failed, msgs, _ = product_reader(path, mode, trims, str(tmp_path / "dump.txt"), capfd)
    assert failed and msgs
    util.assert_matches((failed, msgs, b""), want, case)


def test_arg_desc_lists_the_options():
    out = subprocess.run([CLI, "--arg-desc"], stdout=subprocess.PIPE, check=True).stdout.decode().splitlines()
    for opt in ("phred33", "phred33-quals", "phred64", "phred64-quals", "solexa1.3-quals", "solexa-quals", "int-quals", "integer-quals"):
        assert "%s\t0" % opt in out
