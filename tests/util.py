"""Shared helpers for the test-suite: fixture building, read packing, ctypes bindings of the
oracle (oracle/_ref/libcforacle.so, test infrastructure) and of the host-compiled product
logic (tests/native/hostlogic.cpp), and the recorded outputs of the unmodified reference."""
import atexit
import base64
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import synth  # noqa: E402

REFDIR = os.path.join(ROOT, "oracle", "_ref")
REF_CLASS = os.path.join(REFDIR, "centrifuge-class")
REF_BUILD = os.path.join(REFDIR, "centrifuge-build-bin")
ORACLE_BIN = os.path.join(REFDIR, "cf_oracle")
ORACLE_LIB = os.path.join(REFDIR, "libcforacle.so")
HOSTLOGIC_LIB = os.environ.get("CFB_HOSTLOGIC_LIB", os.path.join(REFDIR, "libhostlogic.so"))   # override: a sanitizer build of the shim
PRODUCT_LIB = os.environ.get("CFB_PRODUCT_LIB", os.path.join(ROOT, "centrifuge_b200", "libcfb200.so"))   # override: sanitizer build of the host side (tests/native/host_stub.cpp)
GOLDEN = os.path.join(ROOT, "tests", "golden")
CACHE = os.environ.get("CFB_TEST_CACHE", os.path.join(tempfile.gettempdir(), "cfb200_test_cache"))

ASC2DNA = np.zeros(256, dtype=np.uint8)
for ch, v in (("A", 0), ("C", 1), ("G", 2), ("T", 3), ("N", 4)):
    ASC2DNA[ord(ch)] = v
    ASC2DNA[ord(ch.lower())] = v


def have_ref():
    return os.path.exists(REF_CLASS) and os.path.exists(REF_BUILD)


# ----------------------------------------------------------------------------- recorded reference outputs
# The differential tests compare with what the unmodified reference (its binaries under oracle/_ref, its Perl scripts in
# its source tree) writes for the same inputs.  Those outputs are recorded as SHA-256 digests in REF_DIGESTS, so that
# the tests run where the reference is not present.  Re-record with the reference built by build() (its sources in
# CFB_REFERENCE_TREE or in a `reference` checkout beside this repository):
#   CFB_RECORD_REFERENCE=1 python -m pytest tests
RECORD = os.environ.get("CFB_RECORD_REFERENCE") == "1"
REF_TREE = os.path.abspath(os.environ.get("CFB_REFERENCE_TREE") or os.path.join(os.path.dirname(ROOT), "reference"))
REF_DIGESTS = os.path.join(GOLDEN, "reference_digests.json")
_digests = None
_recorded = {}


def digest(x):
    """Digest of an output (bytes, str, numbers, booleans, or tuples / lists of them): the first 64 bits of its SHA-256,
    in URL-safe base64."""
    return base64.urlsafe_b64encode(hashlib.sha256(repr(x).encode()).digest()[:8]).decode().rstrip("=")


def assert_matches(got, want, *context):
    """digest(got) == want, a recorded reference digest.  On a mismatch the output is written under CACHE/mismatch/<want>/,
    one file per part, to be compared by hand with the reference's output for the same case."""
    d = digest(got)
    if d == want:
        return
    path = os.path.join(CACHE, "mismatch", want)
    os.makedirs(path, exist_ok=True)
    for i, part in enumerate(got if isinstance(got, (tuple, list)) else (got,)):
        with open(os.path.join(path, "part%d" % i), "wb") as f:
            f.write(part if isinstance(part, bytes) else repr(part).encode())
    raise AssertionError("output (digest %s) differs from the reference's (%s); kept in %s %s" % (d, want, path, context))


def reference(key, run):
    """Digest of what the reference produced for the case named `key`.  run() produces that output with the reference;
    it is called only when recording."""
    global _digests
    if RECORD:
        if not have_ref():
            raise RuntimeError("CFB_RECORD_REFERENCE=1 needs the reference binaries under oracle/_ref (make -C oracle ref)")
        d = digest(run())
        if not _recorded:
            atexit.register(_save_digests)
        _recorded[key] = d
        return d
    if _digests is None:
        with open(REF_DIGESTS) as f:
            _digests = json.load(f)
    if key not in _digests:
        raise KeyError("no recorded reference output for %r (re-record, see tests/util.py)" % key)
    return _digests[key]


def _save_digests():
    old = {}
    if os.path.exists(REF_DIGESTS):
        with open(REF_DIGESTS) as f:
            old = json.load(f)
    old.update(_recorded)
    with open(REF_DIGESTS, "w") as f:
        json.dump(old, f, indent=0, sort_keys=True)
        f.write("\n")


def ref_script(name, tmp):
    """Stage the reference's Perl script `name` (recording only) with the centrifuge-inspect it calls beside it."""
    import shutil
    import stat
    src = os.path.join(REF_TREE, name)
    if not os.path.exists(src):
        raise RuntimeError("recording needs the reference's sources (no %s; set CFB_REFERENCE_TREE)" % src)
    stage = os.path.join(str(tmp), "stage")
    os.makedirs(stage, exist_ok=True)
    shutil.copy(src, os.path.join(stage, name))
    shim = os.path.join(stage, "centrifuge-inspect")
    with open(shim, "w") as f:
        f.write("#!/bin/sh\nexec %s \"$@\"\n" % os.path.join(REFDIR, "centrifuge-inspect-bin"))
    os.chmod(shim, os.stat(shim).st_mode | stat.S_IEXEC)
    return os.path.join(stage, name)


def geometry_args(ftab_chars=10, off_rate=4):
    """centrifuge-build's -t/--ftabchars and -o/--offrate for an index geometry; none for the default (10, 4)."""
    return ([] if ftab_chars == 10 else ["-t", str(ftab_chars)]) + ([] if off_rate == 4 else ["-o", str(off_rate)])


def build_cf(fastas, conv, nodes, names, base, key, ftab_chars=10, off_rate=4):
    """.cf index of the FASTA files: built by the unmodified reference builder when recording, else by the project's own
    GPU builder (cfb_build_index), whose files must equal the reference's (compared by their recorded digest)."""
    def files():
        return [open("%s.%s.cf" % (base, k), "rb").read() for k in "1234"]

    def ref():
        subprocess.check_call([REF_BUILD, "-p", "4", "--conversion-table", conv, "--taxonomy-tree", nodes, "--name-table", names]
                              + geometry_args(ftab_chars, off_rate) + [",".join(fastas), base], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        return files()
    want = reference("index/" + key, ref)
    if not RECORD:
        from centrifuge_b200 import capi
        capi.build_index(capi.build_opts(base, fasta=list(fastas), conversion_table=conv, taxonomy_tree=nodes, name_table=names,
                                         ftab_chars=ftab_chars, off_rate=off_rate))
        if digest(files()) != want:
            raise AssertionError("index %s: the project's builder did not write the reference builder's bytes" % key)


def ensure_oracle():
    """Build the CPU restatement (and the host-logic shim) if missing."""
    if not (os.path.exists(ORACLE_LIB) and os.path.exists(ORACLE_BIN)
            and os.path.getmtime(ORACLE_LIB) >= os.path.getmtime(os.path.join(ROOT, "oracle", "cf_oracle.cpp"))):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "port"], stdout=subprocess.DEVNULL)
    srcs = [os.path.join(ROOT, "tests", "native", "hostlogic.cpp"),
            os.path.join(ROOT, "centrifuge_b200", "csrc", "cf_index.cpp"),
            os.path.join(ROOT, "centrifuge_b200", "csrc", "cf_index.h"),
            os.path.join(ROOT, "centrifuge_b200", "csrc", "cf_logic.h")]
    if not os.path.exists(HOSTLOGIC_LIB) or any(os.path.getmtime(s) > os.path.getmtime(HOSTLOGIC_LIB) for s in srcs):
        os.makedirs(REFDIR, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", HOSTLOGIC_LIB, srcs[0], srcs[1]])


# ----------------------------------------------------------------------------- fixtures
def index_key(tag, genera, species, length, seed, div=0.03, cid=False, strains=False, ftab_chars=10, off_rate=4):
    """Cache directory name of build_index's index, and its recorded digest's key (index/<key>)."""
    args = (tag, genera, species, length, seed, div, cid, strains, tuple(geometry_args(ftab_chars, off_rate)))
    return "%s_%s" % (tag, hashlib.md5(repr(args).encode()).hexdigest()[:12])


def build_index(tag, genera, species, length, seed, div=0.03, cid=False, strains=False, ftab_chars=10, off_rate=4):
    """Synthetic genomes -> .cf index with the reference builder's bytes (build_cf).  Cached.  The builder arguments of a
    non-default geometry go into the key's last field, so the default geometry keeps its key."""
    key = index_key(tag, genera, species, length, seed, div, cid, strains, ftab_chars, off_rate)
    d = os.path.join(CACHE, key)
    base = os.path.join(d, "idx")
    if not os.path.exists(os.path.join(d, "done")):
        os.makedirs(d, exist_ok=True)
        synth.write_genomes(d, genera, species, length, seed, div, cid, strains)
        build_cf([os.path.join(d, "genomes.fa")], os.path.join(d, "conv.tsv"), os.path.join(d, "nodes.dmp"), os.path.join(d, "names.dmp"),
                 base, key, ftab_chars, off_rate)
        open(os.path.join(d, "done"), "w").close()
    return base


def golden_index(name):
    """Decompress a committed golden index (tests/golden/<name>.{1,2,3,4}.cf.xz) into the cache."""
    import lzma
    d = os.path.join(CACHE, "golden")
    os.makedirs(d, exist_ok=True)
    base = os.path.join(d, name)
    for k in "1234":
        dst = "%s.%s.cf" % (base, k)
        src = os.path.join(GOLDEN, "%s.%s.cf.xz" % (name, k))
        if not os.path.exists(dst) or os.path.getmtime(dst) < os.path.getmtime(src):
            with lzma.open(src) as f, open(dst + ".tmp", "wb") as g:
                g.write(f.read())
            os.replace(dst + ".tmp", dst)
    return base


def parse_reads(path):
    """Minimal FASTA/FASTQ reader for tests -> list of (name, uint8 ascii array)."""
    out = []
    with open(path, "rb") as f:
        data = f.read().split(b"\n")
    if not data or not data[0]:
        return out
    if data[0][:1] == b">":
        name, seq = None, []
        for ln in data:
            if ln[:1] == b">":
                if name is not None:
                    out.append((name, np.frombuffer(b"".join(seq), dtype=np.uint8)))
                name, seq = ln[1:].decode(), []
            elif ln:
                seq.append(ln.strip())
        if name is not None:
            out.append((name, np.frombuffer(b"".join(seq), dtype=np.uint8)))
    else:
        for i in range(0, len(data) - 3, 4):
            if data[i][:1] != b"@":
                break
            out.append((data[i][1:].decode(), np.frombuffer(data[i + 1].strip(), dtype=np.uint8)))
    return out


def n_filter_ok(codes):
    """Scoring::nFilter with NCEIL=L,0,0.15 plus the length filter (centrifuge.cpp:2559-2584)."""
    n = len(codes)
    return n >= 2 and int((codes == 4).sum()) <= int(0.15 * n)


class Batch:
    """Packed batch in the C-ABI layout (1 byte/base, 0..4)."""

    def __init__(self, mates1, mates2=None):
        n = len(mates1)
        self.n = n
        self.paired = mates2 is not None
        seqs = [ASC2DNA[a] for a in mates1]
        if self.paired:
            seqs2 = [ASC2DNA[a] for a in mates2]
        self.len1 = np.array([len(s) for s in seqs], dtype=np.uint32)
        self.off1 = np.zeros(n, dtype=np.uint64)
        if n:
            self.off1[1:] = np.cumsum(self.len1[:-1], dtype=np.uint64)
        tot1 = int(self.len1.sum())
        flags = np.array([1 if n_filter_ok(s) else 0 for s in seqs], dtype=np.uint8)
        if self.paired:
            self.len2 = np.array([len(s) for s in seqs2], dtype=np.uint32)
            self.off2 = np.zeros(n, dtype=np.uint64)
            if n:
                self.off2[1:] = np.cumsum(self.len2[:-1], dtype=np.uint64)
            self.off2 += np.uint64(tot1)
            flags |= np.array([2 if n_filter_ok(s) else 0 for s in seqs2], dtype=np.uint8)
            flags |= np.array([4 if len(s) > 0 else 0 for s in seqs2], dtype=np.uint8)   # oracle: bit2 = unit is a pair
            self.bases = np.concatenate(seqs + seqs2) if n else np.zeros(0, dtype=np.uint8)
        else:
            self.len2 = np.zeros(n, dtype=np.uint32)
            self.off2 = np.zeros(n, dtype=np.uint64)
            self.bases = np.concatenate(seqs) if n else np.zeros(0, dtype=np.uint8)
        self.bases = np.ascontiguousarray(self.bases, dtype=np.uint8)
        self.flags = flags


REC = np.dtype([("taxid", "<u8"), ("score", "<u4"), ("hitlen", "<u4"), ("uid", "<u4"), ("pad", "<u4")])


class OParams(C.Structure):
    _fields_ = [("khits", C.c_int), ("min_hitlen", C.c_int), ("tree_traverse", C.c_int), ("class_rank_slot", C.c_int),
                ("host", C.POINTER(C.c_uint64)), ("n_host", C.c_size_t), ("excl", C.POINTER(C.c_uint64)), ("n_excl", C.c_size_t)]


def make_oparams(k=5, min_hitlen=22, traverse=True, rank_slot=0, host=(), excl=()):
    p = OParams()
    p.khits, p.min_hitlen, p.tree_traverse, p.class_rank_slot = k, min_hitlen, 1 if traverse else 0, rank_slot
    p._h = (C.c_uint64 * max(1, len(host)))(*host)
    p._e = (C.c_uint64 * max(1, len(excl)))(*excl)
    p.host, p.n_host = C.cast(p._h, C.POINTER(C.c_uint64)), len(host)
    p.excl, p.n_excl = C.cast(p._e, C.POINTER(C.c_uint64)), len(excl)
    return p


def _ptr(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class _Classifier:
    """Common driver for the oracle and the host-logic shim (identical call signature)."""

    def __init__(self, lib, load, free, classify, base):
        self.lib, self._free, self._classify = lib, free, classify
        err = C.create_string_buffer(256)
        load.restype = C.c_void_p
        self.h = load(base.encode(), err, 256)
        if not self.h:
            raise RuntimeError(err.value.decode())
        classify.restype = C.c_longlong

    def close(self):
        if self.h:
            self._free(C.c_void_p(self.h))
            self.h = None

    def classify(self, batch, params, counters=False):
        n = batch.n
        out_n = np.zeros(n, dtype=np.uint32)
        cap = max(1024, n * 64)
        while True:
            out = np.zeros(cap, dtype=REC)
            ctr = (C.c_uint64 * 16)()
            r = self._classify(C.c_void_p(self.h), C.byref(params), _ptr(batch.bases, C.c_uint8), _ptr(batch.off1, C.c_uint64),
                               _ptr(batch.len1, C.c_uint32), _ptr(batch.off2, C.c_uint64), _ptr(batch.len2, C.c_uint32),
                               _ptr(batch.flags, C.c_uint8), C.c_size_t(n), _ptr(out_n, C.c_uint32),
                               out.ctypes.data_as(C.c_void_p), C.c_size_t(cap), ctr)
            if r == -1:
                cap *= 4
                continue
            if r < 0:
                raise RuntimeError("classify failed: %d" % r)
            return out_n, out[:r], list(ctr)


def Oracle(base):
    ensure_oracle()
    lib = C.CDLL(ORACLE_LIB)
    return _Classifier(lib, lib.cfo_index_load, lib.cfo_index_free, lib.cfo_classify, base)


def HostLogic(base):
    ensure_oracle()
    lib = C.CDLL(HOSTLOGIC_LIB)
    return _Classifier(lib, lib.hl_load, lib.hl_free, lib.hl_classify, base)


ORACLE_STATS = ["reads", "partial_searches", "ftab_probes", "lf_range_steps", "lf_range_same_side", "lf_single_steps",
                "sides_search", "walk_steps", "rows_resolved", "hits_resolved", "ext_searches"]


def run_cli(binary, args, out_tsv, report, env=None):
    subprocess.check_call([binary] + list(args) + ["-S", out_tsv, "--report-file", report],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, env=env)
    with open(out_tsv, "rb") as f:
        a = f.read()
    with open(report, "rb") as f:
        b = f.read()
    return a, b
