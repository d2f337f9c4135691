"""--n-ceil end to end without a GPU: the oracle classifies each input under filter flags from the reference's ceiling,
the product's record-level reader and formatter (cfb_test_host_path_nceil, whose own flags follow the same --n-ceil)
write the TSV, the report and the Kraken-style report, and all three equal what the reference binary wrote for the
same run (recorded digests, tests/golden/n_ceil_digests.json)."""
import ctypes as C
import os

import numpy as np
import pytest

import util
import util_nceil as U


@pytest.fixture(scope="module")
def inputs():
    return U.write_inputs(os.path.join(util.CACHE, "n_ceil_inputs"))


def _units(name):
    """(mate-1 reads, mate-2 reads or None) of an input set, as the reader sees them ('.' is N)"""
    singles, m1, m2 = U.make_reads()
    if name == "pe":
        return m1, m2
    return singles, None


@pytest.mark.parametrize("spec", U.CEILS, ids=U.ceil_key)
@pytest.mark.parametrize("name", ["se", "fa", "pe"])
def test_oracle_and_host_formatter_match_reference(adv_base, inputs, tmp_path, spec, name):
    args = inputs[name]
    want = U.reference("%s/%s" % (name, U.ceil_key(spec)), lambda: U.run_cli(util.REF_CLASS, ["-x", adv_base] + args + U.ceil_args(spec), tmp_path))
    want_kr = U.reference("kreport/%s/%s" % (name, U.ceil_key(spec)), lambda: U.ref_kreport(adv_base, args + U.ceil_args(spec), tmp_path))
    if util.RECORD:
        return
    f = U.PARSED[spec]
    a, b = _units(name)
    enc = lambda s: np.frombuffer(s.replace(".", "N").encode(), dtype=np.uint8)  # noqa: E731
    batch = util.Batch([enc(s) for _, s in a], [enc(s) for _, s in b] if b else None)
    flags = np.array([1 if U.passes(f, s) else 0 for _, s in a], dtype=np.uint8)
    if b:
        flags |= np.array([(2 if U.passes(f, s) else 0) | (4 if s else 0) for _, s in b], dtype=np.uint8)
    batch.flags = flags
    o = util.Oracle(adv_base)
    try:
        n, recs, _ = o.classify(batch, util.make_oparams())
    finally:
        o.close()
    rec_off = np.zeros(len(n) + 1, dtype=np.uint32)
    rec_off[1:] = np.cumsum(n)
    recs = np.ascontiguousarray(recs)
    tsv, rep, kr = (str(tmp_path / x) for x in ("h.tsv", "h.rep", "h.kreport"))
    files = [a_ for a_ in args if a_ not in ("-U", "-1", "-2", "-f")]
    lib = C.CDLL(util.PRODUCT_LIB)
    rc = lib.cfb_test_host_path_nceil(adv_base.encode(), files[0].encode(), files[1].encode() if b else None, C.c_int(1 if name == "fa" else 0),
                                      C.c_int(5), C.c_uint32(0), 0, 0, rec_off.ctypes.data_as(C.POINTER(C.c_uint32)),
                                      recs.ctypes.data_as(C.c_void_p), C.c_uint64(len(n)), None,
                                      spec.encode() if spec is not None else None, tsv.encode(), rep.encode(), kr.encode())
    assert rc == 0
    with open(tsv, "rb") as f1, open(rep, "rb") as f2, open(kr, "rb") as f3:
        util.assert_matches((f1.read(), f2.read()), want, name, spec)
        util.assert_matches(f3.read(), want_kr, name, spec, "kreport")
