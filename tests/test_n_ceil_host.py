"""--n-ceil without a GPU: the shared parser (cf_nceil.h) against the reference binary's verdicts, the ceiling the device
tokeniser evaluates (compiled for the host) against the reference's formula over every length up to 2^20 and sampled
longer ones, the record-level reader's per-read filter verdicts, and the option table."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import util
import util_nceil as U

CLI = os.path.join(util.ROOT, "centrifuge_b200", "centrifuge-class")


@pytest.fixture(scope="module")
def shim():
    src = os.path.join(util.ROOT, "tests", "native", "nceil_host.cpp")
    hdr = os.path.join(util.ROOT, "centrifuge_b200", "csrc", "cf_nceil.h")
    out = os.path.join(util.CACHE, "libnceil_host.so")
    os.makedirs(util.CACHE, exist_ok=True)
    if not os.path.exists(out) or max(os.path.getmtime(src), os.path.getmtime(hdr)) > os.path.getmtime(out):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", out + ".tmp", src])
        os.replace(out + ".tmp", out)
    lib = C.CDLL(out)
    lib.nc_full_cap.restype = C.c_uint32
    return lib


def _eval(shim, f, lens):
    lens = np.ascontiguousarray(lens, dtype=np.uint64)
    out = np.zeros(len(lens), dtype=np.uint64)
    shim.nc_eval_many(C.c_int(f[0]), C.c_double(f[1]), C.c_double(f[2]), lens.ctypes.data_as(C.POINTER(C.c_uint64)),
                      C.c_uint64(len(lens)), out.ctypes.data_as(C.POINTER(C.c_uint64)))
    return out


def _lengths():
    rng = random.Random(3)
    big = [rng.randrange(1 << 20, 1 << 31) for _ in range(20000)] + [(1 << 31) - 1, 8388612, 8388613, 60000, 60001]
    return np.concatenate([np.arange(0, (1 << 20) + 1, dtype=np.uint64), np.array(big, dtype=np.uint64)])


@pytest.mark.parametrize("spec", U.CEILS + [""], ids=U.ceil_key)
def test_parser_matches_reference(shim, spec):
    """the shared parser gives the function the reference parses the option to"""
    if spec is None:
        return
    t, c, l = C.c_int(), C.c_double(), C.c_double()
    err = C.create_string_buffer(256)
    assert shim.nc_parse(spec.encode(), C.byref(t), C.byref(c), C.byref(l), err, 256) == 0, err.value
    assert (t.value, c.value, l.value) == U.PARSED[spec]


@pytest.mark.parametrize("spec", U.BAD_CEILS)
def test_refused_values_match_reference(spec):
    """exit code and first stderr line of a refused --n-ceil value, as the reference binary prints them"""
    want = U.reference("error/[%s]" % spec, lambda: U.error_of(util.REF_CLASS, spec))
    got = U.error_of(CLI, spec)
    util.assert_matches(got, want, spec)


@pytest.mark.parametrize("spec", U.CEILS, ids=U.ceil_key)
def test_device_formula_equals_reference_formula(shim, spec):
    """nceil_eval (what k_tok_bases runs, built for the host) equals SimpleFunc::f<size_t> restated in Python floats"""
    f = U.PARSED[spec]
    lens = _lengths()
    got = _eval(shim, f, lens)
    if f[0] == 2:                       # linear: vectorised restatement (IEEE multiply and add; these ceilings stay below 2^63)
        t, c, l = f
        v = c + l * lens.astype(np.float64)
        assert np.array_equal(got, np.where(0.0 < v, v, 0.0).astype(np.uint64))
    elif f[0] == 1:                     # constant: one value
        assert (got == np.uint64(U.ceiling(f, 0))).all()
    else:
        want = np.array([U.ceiling(f, int(n)) for n in lens], dtype=np.uint64)
        assert np.array_equal(got, want)
    if spec is None:                    # the default decides as the literal it replaces in the tokeniser and the reader
        small = lens[lens < (1 << 32)]
        assert np.array_equal(got[: len(small)], (0.15 * small.astype(np.float64)).astype(np.uint32).astype(np.uint64))


def test_ceiling_edge_cases(shim):
    """G at lengths 0 and 1, a negative ceiling, ceilings past the length, 2^63 and past 2^64"""
    g = _eval(shim, (4, 0.0, 3.0), [0, 1, 2, 3])
    assert list(g) == [0, 0, 2, 3]                                    # ln 0 = -inf -> 0; ln 1 = 0
    assert list(_eval(shim, (4, 2.0, 0.0), [0, 1])) == [2 ** 64 - 1, 2]   # 0 * -inf is NaN: min(X, NaN) = X = DBL_MAX
    assert list(_eval(shim, (1, -3.0, 0.0), [0, 5, 100])) == [0, 0, 0]
    assert list(_eval(shim, (1, 1e9, 0.0), [10])) == [10 ** 9]
    assert list(_eval(shim, (1, 2.0 ** 63, 0.0), [10])) == [2 ** 63]
    assert list(_eval(shim, (1, 1e30, 0.0), [10])) == [0]             # (size_t) of a double past 2^64 on x86-64
    assert list(_eval(shim, (1, 1.7976931348623157e308, 0.0), [10])) == [2 ** 64 - 1]


def test_unset_coefficient_is_the_reference_float(shim):
    """`S,<c>`, `L,<c>` and `G,<c>` keep the policy's 0.15f coefficient: at the lengths where 0.15f and 0.15 part the
    ceiling is the reference's, and a parsed L,0,0.15 (the double) keeps the product's default"""
    t, c, l = C.c_int(), C.c_double(), C.c_double()
    err = C.create_string_buffer(256)
    for spec, n in (("S,1", 1504711), ("L,0", 8388613), ("G,2", 485164810)):
        assert shim.nc_parse(spec.encode(), C.byref(t), C.byref(c), C.byref(l), err, 256) == 0
        f = (t.value, c.value, l.value)
        assert l.value == U.F15
        got = int(_eval(shim, f, [n])[0])
        assert got == U.ceiling(f, n) != U.ceiling((f[0], f[1], 0.15), n), spec
    assert shim.nc_parse(b"L,0,0.15", C.byref(t), C.byref(c), C.byref(l), err, 256) == 0 and l.value == 0.15


def test_full_cap_follows_the_ceiling(shim):
    """the hit-list bound grows with the ceiling, stays at the default's for small ceilings, and never passes len + 2"""
    for maxlen in (128, 160, 320, 1024, 60000):
        assert shim.nc_full_cap(2, C.c_double(0.0), C.c_double(0.15), maxlen) == maxlen // 4 + 8
        assert shim.nc_full_cap(1, C.c_double(0.0), C.c_double(0.15), maxlen) == maxlen // 4 + 8
        assert shim.nc_full_cap(2, C.c_double(0.0), C.c_double(1.0), maxlen) == maxlen + 2
        assert shim.nc_full_cap(1, C.c_double(1e30), C.c_double(0.0), maxlen) == maxlen // 4 + 8


@pytest.mark.parametrize("spec", U.CEILS, ids=U.ceil_key)
def test_record_reader_verdicts(tmp_path, spec):
    """cfb_test_parse_nceil's per-read N-filter verdicts equal the reference's nFilter + lenfilt restated in Python"""
    lib = C.CDLL(util.PRODUCT_LIB)
    d = os.path.join(util.CACHE, "n_ceil_inputs")
    U.write_inputs(d)
    singles, m1, m2 = U.make_reads()
    f = U.PARSED[spec]
    for name, reads, fa in (("se.fq", singles, 0), ("se.fa", singles, 1), ("p2.fq", m2, 0)):
        out = str(tmp_path / "v.txt")
        rc = lib.cfb_test_parse_nceil(os.path.join(d, name).encode(), C.c_int(fa), 0, 0, C.c_uint32(0),
                                      spec.encode() if spec is not None else None, out.encode())
        assert rc == 0
        rows = [ln.split("\t") for ln in open(out).read().splitlines()]
        assert len(rows) == len(reads)
        got = [int(r[3]) for r in rows]
        want = [1 if U.passes(f, r[1]) else 0 for r in rows]          # the reader's own bases: '.' read as N
        assert got == want, name
        assert sum(got) > 0


def test_arg_desc_lists_the_options():
    out = subprocess.run([CLI, "--arg-desc"], stdout=subprocess.PIPE, check=True).stdout.decode().splitlines()
    for opt, arg in (("n-ceil", 1), ("ignore-quals", 0), ("nofw", 0), ("norc", 0)):
        assert "%s\t%d" % (opt, arg) in out


@pytest.mark.parametrize("flags", U.QUIRK_FLAGS, ids=lambda f: "+".join(x.strip("-") for x in f))
def test_quirk_flags_change_nothing_in_the_reference(flags):
    """--ignore-quals, --nofw and --norc leave the reference's output as it is (recorded digests equal)"""
    base = U.reference("se/default", None) if not util.RECORD else None
    if util.RECORD:
        pytest.skip("compared after recording")
    assert U.reference("se/default/" + "+".join(flags), None) == base
