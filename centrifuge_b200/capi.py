"""ctypes binding of include/cfb200.h (the C ABI of libcfb200.so).

Python is plumbing only: every call below lands in the CUDA library.  There is no CPU
fallback -- loading the library or creating a context without a usable sm_90 (H100) device raises.
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcfb200.so")

CFB_UID_NONE = 0xFFFFFFFF
REC_DTYPE = np.dtype([("taxid", "<u8"), ("score", "<u4"), ("hitlen", "<u4"), ("uid", "<u4"), ("pad", "<u4")])

_lib = None


class CfbError(RuntimeError):
    pass


class IndexInfo(C.Structure):
    _fields_ = [("len", C.c_uint64), ("num_sides", C.c_uint64), ("n_seqs", C.c_uint64), ("n_tax_nodes", C.c_uint64),
                ("n_boundaries", C.c_uint64), ("line_rate", C.c_int32), ("off_rate", C.c_int32), ("ftab_chars", C.c_int32),
                ("sample_bytes", C.c_int32), ("compressed", C.c_int32), ("device", C.c_int32), ("device_bytes", C.c_uint64)]


class IndexTables(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("sides_bytes", "sample_bytes", "rank16_bytes", "ftab2_bytes", "ftabk_bytes", "resolve_table_bytes",
                                          "walk8_bytes", "total_bytes", "free_bytes_after_load", "walk8_rows", "ftabd_bytes")] + [("ftabk_chars", C.c_int32), ("resolve_entry_bytes", C.c_int32), ("ftabd_chars", C.c_int32), ("pad", C.c_int32)]


class Params(C.Structure):
    _fields_ = [("khits", C.c_int32), ("min_hitlen", C.c_int32), ("tree_traverse", C.c_int32), ("class_rank_slot", C.c_int32),
                ("host_taxids", C.POINTER(C.c_uint64)), ("n_host_taxids", C.c_uint64),
                ("excluded_taxids", C.POINTER(C.c_uint64)), ("n_excluded_taxids", C.c_uint64)]


class BatchC(C.Structure):
    _fields_ = [("n_units", C.c_uint64), ("n_mates", C.c_int32), ("bases", C.POINTER(C.c_uint8)), ("n_bases", C.c_uint64),
                ("off", C.POINTER(C.c_uint64) * 2), ("len", C.POINTER(C.c_uint32) * 2), ("flags", C.POINTER(C.c_uint8))]


class BatchPackedC(C.Structure):
    _fields_ = [("n_units", C.c_uint64), ("n_mates", C.c_int32), ("words", C.POINTER(C.c_uint64)), ("n_words", C.c_uint64),
                ("len", C.POINTER(C.c_uint32) * 2), ("n_pos", C.POINTER(C.c_uint64)), ("n_n", C.c_uint64), ("flags", C.POINTER(C.c_uint8))]


class ResultC(C.Structure):
    _fields_ = [("n_units", C.c_uint64), ("n_recs", C.c_uint64), ("rec_off", C.POINTER(C.c_uint32)), ("recs", C.c_void_p)]


def lib():
    """Load libcfb200.so (building nothing: run centrifuge_b200.build first)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CfbError("libcfb200.so is not built (python -m centrifuge_b200.build); there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        L.cfb_last_error.restype = C.c_char_p
        L.cfb_version.restype = C.c_char_p
        L.cfb_index_seq_name.restype = C.c_char_p
        L.cfb_index_seq_taxid.restype = C.c_uint64
        L.cfb_host_alloc.restype = C.c_void_p
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise CfbError("cfb200 error %d: %s" % (rc, lib().cfb_last_error().decode()))


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Index:
    def __init__(self, basename, device=0, flags=0):
        self.h = C.c_void_p()
        _ck(lib().cfb_index_load_ex(basename.encode(), C.c_int(device), C.c_uint32(flags), C.byref(self.h)))
        self.info = IndexInfo()
        _ck(lib().cfb_index_get_info(self.h, C.byref(self.info)))

    def tables(self):
        """dict of what the device replica holds (cfb_index_get_tables)"""
        t = IndexTables()
        _ck(lib().cfb_index_get_tables(self.h, C.byref(t)))
        return {n: int(getattr(t, n)) for n, _ in IndexTables._fields_}

    def seq_name(self, i):
        s = lib().cfb_index_seq_name(self.h, C.c_uint32(i))
        return s.decode() if s is not None else None

    def seq_taxid(self, i):
        return int(lib().cfb_index_seq_taxid(self.h, C.c_uint32(i)))

    def tax_node(self, taxid):
        par, rank, leaf = C.c_uint64(), C.c_int(), C.c_int()
        ok = lib().cfb_index_tax_node(self.h, C.c_uint64(taxid), C.byref(par), C.byref(rank), C.byref(leaf))
        return (int(par.value), rank.value, leaf.value) if ok else None

    def node_taxids(self):
        n = int(self.info.n_tax_nodes)
        out = np.zeros(n, dtype=np.uint64)
        _ck(lib().cfb_index_node_taxids(self.h, _p(out, C.c_uint64), C.c_uint64(n)))
        return out

    def close(self):
        if self.h:
            lib().cfb_index_free(self.h)
            self.h = C.c_void_p()


def make_params(k=5, min_hitlen=22, traverse=True, rank_slot=0, host=(), excl=()):
    p = Params()
    lib().cfb_params_default(C.byref(p))
    p.khits, p.min_hitlen, p.tree_traverse, p.class_rank_slot = k, min_hitlen, 1 if traverse else 0, rank_slot
    p._h = (C.c_uint64 * max(1, len(host)))(*host)
    p._e = (C.c_uint64 * max(1, len(excl)))(*excl)
    p.host_taxids, p.n_host_taxids = C.cast(p._h, C.POINTER(C.c_uint64)), len(host)
    p.excluded_taxids, p.n_excluded_taxids = C.cast(p._e, C.POINTER(C.c_uint64)), len(excl)
    return p


def make_batch(bases, off1, len1, off2=None, len2=None, flags=None):
    """numpy arrays -> BatchC (keeps references alive on the returned object)."""
    b = BatchC()
    b.n_units = len(len1)
    b.n_mates = 2 if off2 is not None else 1
    b.bases, b.n_bases = _p(bases, C.c_uint8), bases.size
    b.off[0], b.len[0] = _p(off1, C.c_uint64), _p(len1, C.c_uint32)
    if off2 is not None:
        b.off[1], b.len[1] = _p(off2, C.c_uint64), _p(len2, C.c_uint32)
    if flags is not None:
        b.flags = _p(flags, C.c_uint8)
    b._keep = (bases, off1, len1, off2, len2, flags)
    return b


def make_batch_packed(words, len1, len2=None, n_pos=None, flags=None):
    b = BatchPackedC()
    b.n_units = len(len1)
    b.n_mates = 2 if len2 is not None else 1
    b.words, b.n_words = _p(words, C.c_uint64), words.size
    b.len[0] = _p(len1, C.c_uint32)
    if len2 is not None:
        b.len[1] = _p(len2, C.c_uint32)
    if n_pos is not None and n_pos.size:
        b.n_pos, b.n_n = _p(n_pos, C.c_uint64), n_pos.size
    if flags is not None:
        b.flags = _p(flags, C.c_uint8)
    b._keep = (words, len1, len2, n_pos, flags)
    return b


def pack_batch(batch):
    """cfb_pack_batch: (words, n_pos) of a byte-form BatchC"""
    nw, nn = C.c_uint64(), C.c_uint64()
    lib().cfb_pack_batch(C.byref(batch), None, C.c_uint64(0), None, C.c_uint64(0), C.byref(nw), C.byref(nn))
    words = np.zeros(max(1, int(nw.value)), dtype=np.uint64); npos = np.zeros(max(1, int(nn.value)), dtype=np.uint64)
    _ck(lib().cfb_pack_batch(C.byref(batch), _p(words, C.c_uint64), C.c_uint64(words.size), _p(npos, C.c_uint64), C.c_uint64(npos.size), C.byref(nw), C.byref(nn)))
    return words[:int(nw.value)], npos[:int(nn.value)]


def pack_fixed(codes):
    """vectorised packing of an (n, L) code matrix (0..4): words (n * ceil(L/32),) and the N position list"""
    n, L = codes.shape
    W = (L + 31) // 32
    pad = np.zeros((n, W * 32), dtype=np.uint64)
    isn = codes > 3
    pad[:, :L] = np.where(isn, 0, codes)
    sh = (np.arange(32, dtype=np.uint64) * np.uint64(2))[None, None, :]
    words = (pad.reshape(n, W, 32) << sh).sum(axis=2, dtype=np.uint64).reshape(-1)
    r, j = np.nonzero(isn)
    npos = ((r.astype(np.uint64) * np.uint64(W) + (j // 32).astype(np.uint64)) << np.uint64(5)) | (j % 32).astype(np.uint64)
    return np.ascontiguousarray(words), np.ascontiguousarray(npos)


def pinned_array(shape, dtype):
    """numpy array backed by cfb_host_alloc (pinned) memory: H2D copies are DMA'd straight from it."""
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) * dt.itemsize
    ptr = lib().cfb_host_alloc(C.c_size_t(max(n, 1)))
    if not ptr:
        raise CfbError("cfb_host_alloc failed")
    buf = (C.c_char * max(n, 1)).from_address(ptr)
    a = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
    return a


def _result(res):
    n = int(res.n_units)
    nrec = int(res.n_recs)
    if n == 0:
        return np.zeros(1, dtype=np.uint32), np.zeros(0, dtype=REC_DTYPE)
    off = np.ctypeslib.as_array(res.rec_off, shape=(n + 1,)).copy()
    if nrec:
        buf = (C.c_char * (nrec * REC_DTYPE.itemsize)).from_address(res.recs)
        recs = np.frombuffer(buf, dtype=REC_DTYPE).copy()
    else:
        recs = np.zeros(0, dtype=REC_DTYPE)
    return off, recs


class TextOpts(C.Structure):
    _fields_ = [("fasta", C.c_int32), ("trim5", C.c_int32), ("trim3", C.c_int32), ("seed", C.c_uint32), ("maxlen_hint", C.c_uint32)]


class TextResultC(C.Structure):
    _fields_ = [("n_units", C.c_uint64), ("irregular", C.c_int32), ("maxlen", C.c_uint32), ("tsv", C.c_void_p), ("tsv_bytes", C.c_uint64),
                ("multi", C.POINTER(C.c_uint64)), ("n_multi", C.c_uint64), ("multi_stride", C.c_uint32)]


class Context:
    def __init__(self, index, params=None):
        self.index = index
        self.params = params if params is not None else make_params()
        self.h = C.c_void_p()
        _ck(lib().cfb_ctx_create(index.h, C.byref(self.params), C.byref(self.h)))
        self.n_slots = lib().cfb_ctx_slots(self.h)

    def classify(self, batch):
        res = ResultC()
        _ck(lib().cfb_classify_batch(self.h, C.byref(batch), C.byref(res)))
        return _result(res)

    def submit(self, slot, batch):
        _ck(lib().cfb_classify_submit(self.h, C.c_int(slot), C.byref(batch)))

    def submit_packed(self, slot, pbatch):
        _ck(lib().cfb_classify_submit_packed(self.h, C.c_int(slot), C.byref(pbatch)))

    def wait(self, slot, copy=True):
        res = ResultC()
        _ck(lib().cfb_classify_wait(self.h, C.c_int(slot), C.byref(res)))
        return _result(res) if copy else (int(res.n_units), int(res.n_recs))

    def upload(self, batch):
        d = C.c_void_p()
        _ck(lib().cfb_batch_upload(self.h, C.byref(batch), C.byref(d)))
        return d

    def classify_resident(self, dbatch, first=None, count=None):
        ms = (C.c_float * 5)()
        nrec = C.c_uint64()
        if first is None:
            _ck(lib().cfb_classify_resident(self.h, dbatch, ms, C.byref(nrec)))
        else:
            _ck(lib().cfb_classify_resident_range(self.h, dbatch, C.c_uint64(first), C.c_uint64(count), ms, C.byref(nrec)))
        return list(ms), int(nrec.value)

    def resident_result(self):
        res = ResultC()
        _ck(lib().cfb_resident_result(self.h, C.byref(res)))
        return _result(res)

    def set_columns(self, cols=None):
        """Columns of the rows of later text_submit calls: a --tab-fmt-cols list ("readID,taxID,readSeq,..."); None = the
        default list.  An unknown name raises CfbError with the reference's message."""
        _ck(lib().cfb_ctx_set_columns(self.h, cols.encode() if cols is not None else None))

    def set_n_ceil(self, type_, constant, coeff, min_=0.0, max_=sys.float_info.max):
        """N ceiling of later text_submit calls (--n-ceil): type_ 1 = constant, 2 = linear, 3 = sqrt, 4 = log."""
        _ck(lib().cfb_ctx_set_n_ceil(self.h, C.c_int(type_), C.c_double(constant), C.c_double(coeff), C.c_double(min_), C.c_double(max_)))

    def set_quals(self, solexa=False, phred64=False, integer=False):
        """Quality encoding of later text_submit calls (--solexa-quals, --phred64, --int-quals; all False: phred33)."""
        _ck(lib().cfb_ctx_set_quals(self.h, C.c_int(int(solexa)), C.c_int(int(phred64)), C.c_int(int(integer))))

    def text_submit(self, slot, text_a, text_b=None, n_records=0, fasta=False, trim5=0, trim3=0, seed=0, maxlen_hint=0):
        """text_a/text_b: uint8 arrays of complete records (pinned arrays are DMA'd in place)."""
        o = TextOpts(1 if fasta else 0, trim5, trim3, seed, maxlen_hint)
        pb = _p(text_b, C.c_uint8) if text_b is not None else None
        _ck(lib().cfb_text_submit(self.h, C.c_int(slot), _p(text_a, C.c_uint8), C.c_uint64(text_a.size), pb,
                                  C.c_uint64(text_b.size if text_b is not None else 0), C.c_uint64(n_records), C.byref(o)))

    def text_wait(self, slot, discard=False, copy=True):
        r = TextResultC()
        _ck(lib().cfb_text_wait(self.h, C.c_int(slot), C.c_int(1 if discard else 0), C.byref(r)))
        out = dict(n_units=int(r.n_units), irregular=int(r.irregular), maxlen=int(r.maxlen), tsv_bytes=int(r.tsv_bytes), n_multi=int(r.n_multi))
        if copy and not r.irregular:
            out["tsv"] = C.string_at(r.tsv, r.tsv_bytes) if r.tsv_bytes else b""
            st = int(r.multi_stride)
            out["multi"] = np.ctypeslib.as_array(r.multi, shape=(int(r.n_multi), st)).copy() if r.n_multi else np.zeros((0, st), dtype=np.uint64)
        return out

    def text_species(self):
        n = C.c_uint64()
        _ck(lib().cfb_text_species(self.h, None, None, None, None, C.c_uint64(0), C.byref(n)))
        k = int(n.value)
        arrs = [np.zeros(k, dtype=np.uint64) for _ in range(4)]
        if k:
            _ck(lib().cfb_text_species(self.h, *[_p(a, C.c_uint64) for a in arrs], C.c_uint64(k), C.byref(n)))
        return dict(taxid=arrs[0], n_reads=arrs[1], n_unique=arrs[2], n_obs1=arrs[3])

    # ---- per-taxon counters and the multi-GPU reduction
    def count_records(self, on=True):
        _ck(lib().cfb_ctx_count_records(self.h, C.c_int(1 if on else 0)))

    def counts_taxids(self):
        n = C.c_uint64()
        _ck(lib().cfb_counts_taxids(self.h, None, C.c_uint64(0), C.byref(n)))
        out = np.zeros(int(n.value), dtype=np.uint64)
        _ck(lib().cfb_counts_taxids(self.h, _p(out, C.c_uint64), C.c_uint64(len(out)), C.byref(n)))
        return out

    def counts_reset(self):
        _ck(lib().cfb_counts_reset(self.h))

    def counts_dense(self, global_=False, n=None):
        """(3, n) uint64: numReads, numUniqueReads, observed singletons per entry of counts_taxids()"""
        if n is None:
            n = len(self.counts_taxids())
        out = np.zeros(3 * n, dtype=np.uint64)
        _ck(lib().cfb_counts_dense(self.h, C.c_int(1 if global_ else 0), _p(out, C.c_uint64), C.c_uint64(out.size)))
        return out.reshape(3, n)

    def comm_init_rank(self, nranks, rank, uid):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(uid))
        _ck(lib().cfb_comm_init_rank(self.h, C.c_int(nranks), C.c_int(rank), buf))

    def counts_allreduce(self, out=None):
        """collective over the communicator this context belongs to (a no-op copy without one)"""
        arr = (C.c_void_p * 1)(self.h)
        _ck(lib().cfb_counts_allreduce(arr, C.c_int(1), _p(out, C.c_uint64) if out is not None else None, C.c_uint64(out.size if out is not None else 0)))

    def requests(self):
        out = (C.c_uint64 * 5)()
        _ck(lib().cfb_ctx_requests(self.h, out))
        return dict(zip(["rank16", "ftab2", "ftabk", "walk8", "ftabd"], [int(x) for x in out]))

    def request_breakdown(self):
        """where the CFB_COUNT=2 requests of the last batch go: rank16 requests by range width, walk8 jumps tried / taken"""
        out = (C.c_uint64 * 8)()
        _ck(lib().cfb_ctx_request_breakdown(self.h, out))
        names = ["rank16_w1", "rank16_w2_4", "rank16_w5", "walk8_try_row", "walk8_ok_row", "walk8_try_range", "walk8_ok_range", "walk8_ok_w5"]
        return dict(zip(names, [int(x) for x in out]))

    def search_iter_stats(self):
        """how k_search_t's loop spent its trips in the last batch (CFB_COUNT=2); clocks are SM cycles summed over one lane per warp"""
        out = (C.c_uint64 * 8)()
        _ck(lib().cfb_ctx_search_iter_stats(self.h, out))
        names = ["warp_iters", "lane_requests", "consumer_paths", "restart_paths", "task_iters", "clk_head", "clk_wait", "clk_tail"]
        return dict(zip(names, [int(x) for x in out]))

    def score_stats(self):
        """how k_score spent the last batch (CFB_COUNT=1 or 2): totals, and units by rows / by distinct ids in log2 buckets"""
        out = (C.c_uint64 * 23)()
        _ck(lib().cfb_ctx_score_stats(self.h, out))
        v = [int(x) for x in out]
        names = ["units", "rows", "distinct_ids", "reduce_units", "reduce_rounds", "warps", "warps_global"]
        d = dict(zip(names, v[:7]))
        d["rows_hist"], d["distinct_ids_hist"] = v[7:15], v[15:23]
        return d

    def long_stats(self):
        """long units classified by this context so far (cfb_ctx_long_stats)"""
        out = (C.c_uint64 * 4)()
        _ck(lib().cfb_ctx_long_stats(self.h, out))
        return dict(zip(["units", "bases", "segment_searches", "researched"], [int(x) for x in out]))

    def counters(self):
        out = (C.c_uint64 * 8)()
        _ck(lib().cfb_ctx_counters(self.h, out))
        names = ["units", "partial_searches", "ftab_probes", "sides_search", "walk_steps", "rows_resolved", "lf_steps", "ext_searches"]
        return dict(zip(names, [int(x) for x in out]))

    def launches(self):
        n = C.c_uint64()
        _ck(lib().cfb_ctx_kernel_launches(self.h, C.byref(n)))
        return int(n.value)

    def close(self):
        if self.h:
            lib().cfb_ctx_destroy(self.h)
            self.h = C.c_void_p()


def comm_unique_id():
    buf = (C.c_uint8 * 128)()
    _ck(lib().cfb_comm_unique_id(buf))
    return bytes(buf)


def comm_init_all(contexts):
    arr = (C.c_void_p * len(contexts))(*[c.h for c in contexts])
    _ck(lib().cfb_comm_init_all(arr, C.c_int(len(contexts))))


def counts_allreduce_all(contexts):
    arr = (C.c_void_p * len(contexts))(*[c.h for c in contexts])
    _ck(lib().cfb_counts_allreduce(arr, C.c_int(len(contexts)), None, C.c_uint64(0)))


def gather_ceiling(index, table, n_requests=1 << 30):
    """G requests/s of independent random gathers over one of the replica's arrays (0 rank16, 1 K-mer table, 2 walk8, 3 resolve table)"""
    g, ms = C.c_double(), C.c_double()
    _ck(lib().cfb_gather_ceiling(index.h, C.c_int(table), C.c_uint64(n_requests), C.byref(g), C.byref(ms)))
    return float(g.value), float(ms.value)


def gather_rate(index, table, n_requests, ctas_per_sm, ilp):
    """the gather_ceiling probe with ctas_per_sm x 128 x ilp requests in flight per SM (the ceiling itself is 16, 4)"""
    g, ms = C.c_double(), C.c_double()
    _ck(lib().cfb_gather_rate(index.h, C.c_int(table), C.c_uint64(n_requests), C.c_int(ctas_per_sm), C.c_int(ilp), C.byref(g), C.byref(ms)))
    return float(g.value), float(ms.value)


def test_lf(index, rows, chars):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    chars = np.ascontiguousarray(chars, dtype=np.uint8)
    out = np.zeros(len(rows), dtype=np.uint64)
    _ck(lib().cfb_test_lf(index.h, _p(rows, C.c_uint64), _p(chars, C.c_uint8), C.c_uint64(len(rows)), _p(out, C.c_uint64)))
    return out


def test_resolve(index, rows):
    rows = np.ascontiguousarray(rows, dtype=np.uint64)
    out = np.zeros(len(rows), dtype=np.uint32)
    _ck(lib().cfb_test_resolve(index.h, _p(rows, C.c_uint64), C.c_uint64(len(rows)), _p(out, C.c_uint32)))
    return out


CFB_EDATA = -7


class GunzipState(C.Structure):
    _fields_ = [("in_offset", C.c_uint64), ("out_offset", C.c_uint64), ("bit", C.c_uint64), ("hdr_bit", C.c_uint64),
                ("member_bytes", C.c_uint64), ("crc", C.c_uint32), ("win_len", C.c_uint32), ("phase", C.c_int32),
                ("members", C.c_uint32), ("window", C.c_uint8 * 32768)]


class Gunzip:
    """Streaming gzip inflater on a device (cfb_gunzip_*).  run() takes compressed bytes and returns
    (decompressed bytes, compressed bytes consumed); errors raise CfbError with the code in .code."""

    def __init__(self, device=0, chunk_kb=0):
        self.h = C.c_void_p()
        _ck(lib().cfb_gunzip_create(C.c_int(device), C.c_uint32(chunk_kb), C.byref(self.h)))

    def run(self, data, is_last, out_cap=1 << 24):
        src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        out = np.empty(max(1, out_cap), dtype=np.uint8)
        n_out, n_in = C.c_uint64(), C.c_uint64()
        rc = lib().cfb_gunzip_run(self.h, src.ctypes.data_as(C.c_void_p), C.c_uint64(len(data)), C.c_int(1 if is_last else 0),
                                  out.ctypes.data_as(C.c_void_p), C.c_uint64(out_cap), C.byref(n_out), C.byref(n_in))
        if rc != 0:
            e = CfbError("cfb200 error %d: %s" % (rc, lib().cfb_last_error().decode()))
            e.code = rc
            raise e
        return out[: n_out.value].tobytes(), int(n_in.value)

    def decompress_iter(self, data, piece=None, out_cap=1 << 24):
        """Yield the decompressed stream of `data`, fed in pieces of `piece` bytes (all at once when None)."""
        piece = piece or max(1, len(data))
        pos, held = 0, b""
        while True:
            if pos < len(data) and len(held) < piece:
                held += data[pos: pos + piece]
                pos = min(len(data), pos + piece)
            out, used = self.run(held, pos >= len(data), out_cap)
            held = held[used:]
            if out:
                yield out
            elif not used:
                if pos >= len(data):
                    return
                held += data[pos: pos + piece]             # the inflater needs more input than it holds
                pos = min(len(data), pos + piece)

    def decompress(self, data, piece=None, out_cap=1 << 24):
        return b"".join(self.decompress_iter(data, piece, out_cap))

    def state(self):
        s = GunzipState()
        _ck(lib().cfb_gunzip_get_state(self.h, C.byref(s)))
        return s

    def set_state(self, s):
        _ck(lib().cfb_gunzip_set_state(self.h, C.byref(s)))

    def stats(self):
        st = (C.c_uint64 * 5)()
        _ck(lib().cfb_gunzip_stats(self.h, st))
        return dict(zip(("members", "bytes_in", "bytes_out", "chunks", "redone"), (int(x) for x in st)))

    def close(self):
        if self.h:
            lib().cfb_gunzip_destroy(self.h)
            self.h = C.c_void_p()


class Bunzip2:
    """Streaming bzip2 decompressor on a device (cfb_bunzip2_*).  run() takes compressed bytes and returns
    (decompressed bytes, compressed bytes consumed); errors raise CfbError with the code in .code."""

    def __init__(self, device=0, pass_kb=0):
        self.h = C.c_void_p()
        _ck(lib().cfb_bunzip2_create(C.c_int(device), C.c_uint32(pass_kb), C.byref(self.h)))

    def run(self, data, is_last, out_cap=1 << 24):
        src = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
        out = np.empty(max(1, out_cap), dtype=np.uint8)
        n_out, n_in = C.c_uint64(), C.c_uint64()
        rc = lib().cfb_bunzip2_run(self.h, src.ctypes.data_as(C.c_void_p), C.c_uint64(len(data)), C.c_int(1 if is_last else 0),
                                   out.ctypes.data_as(C.c_void_p), C.c_uint64(out_cap), C.byref(n_out), C.byref(n_in))
        if rc != 0:
            e = CfbError("cfb200 error %d: %s" % (rc, lib().cfb_last_error().decode()))
            e.code = rc
            raise e
        return out[: n_out.value].tobytes(), int(n_in.value)

    def decompress_iter(self, data, piece=None, out_cap=1 << 24):
        """Yield the decompressed stream of `data`, fed in pieces of `piece` bytes (all at once when None)."""
        piece = piece or max(1, len(data))
        pos, held = 0, b""
        while True:
            if pos < len(data) and len(held) < piece:
                held += data[pos: pos + piece]
                pos = min(len(data), pos + piece)
            out, used = self.run(held, pos >= len(data), out_cap)
            held = held[used:]
            if out:
                yield out
            elif not used:
                if pos >= len(data):
                    return
                held += data[pos: pos + piece]             # the decompressor needs more input than it holds
                pos = min(len(data), pos + piece)

    def decompress(self, data, piece=None, out_cap=1 << 24):
        return b"".join(self.decompress_iter(data, piece, out_cap))

    def stats(self):
        st = (C.c_uint64 * 6)()
        _ck(lib().cfb_bunzip2_stats(self.h, st))
        return dict(zip(("streams", "bytes_in", "bytes_out", "blocks", "rejected", "trailing"), (int(x) for x in st)))

    def close(self):
        if self.h:
            lib().cfb_bunzip2_destroy(self.h)
            self.h = C.c_void_p()


class BuildOpts(C.Structure):
    _fields_ = [("out_base", C.c_char_p), ("fasta", C.POINTER(C.c_char_p)), ("n_fasta", C.c_int32),
                ("synth_genera", C.c_uint32), ("synth_species", C.c_uint32), ("synth_len", C.c_uint64), ("synth_seed", C.c_uint64),
                ("synth_div", C.c_double), ("conversion_table", C.c_char_p), ("taxonomy_tree", C.c_char_p), ("name_table", C.c_char_p),
                ("size_table", C.c_char_p), ("ftab_chars", C.c_int32), ("off_rate", C.c_int32), ("device", C.c_int32), ("verbose", C.c_int32),
                ("synth_prefix", C.c_char_p)]


def build_opts(out_base=None, fasta=(), synth=None, conversion_table=None, taxonomy_tree=None, name_table=None, size_table=None,
               ftab_chars=10, off_rate=4, device=0, verbose=0, synth_prefix=None):
    """synth = (genera, species, len, seed, div) for counter-based synthetic genomes."""
    o = BuildOpts()
    lib().cfb_build_opts_default(C.byref(o))
    o.out_base = out_base.encode() if out_base else None
    if fasta:
        o._fa = (C.c_char_p * len(fasta))(*[f.encode() for f in fasta])
        o.fasta, o.n_fasta = C.cast(o._fa, C.POINTER(C.c_char_p)), len(fasta)
    if synth:
        o.synth_genera, o.synth_species, o.synth_len, o.synth_seed, o.synth_div = synth
    for k, v in (("conversion_table", conversion_table), ("taxonomy_tree", taxonomy_tree), ("name_table", name_table), ("size_table", size_table)):
        if v:
            setattr(o, k, v.encode())
    o.ftab_chars, o.off_rate, o.device, o.verbose = ftab_chars, off_rate, device, verbose
    if synth_prefix:
        o.synth_prefix = synth_prefix.encode()
    return o


def build_index(opts):
    L = lib()
    L.cfb_build_last_error.restype = C.c_char_p
    rc = L.cfb_build_index(C.byref(opts))
    if rc != 0:
        raise CfbError("cfb_build_index error %d: %s" % (rc, L.cfb_build_last_error().decode()))


def synth_reads(opts, n, rdlen, seed):
    out = np.zeros((n, rdlen), dtype=np.uint8)
    L = lib()
    L.cfb_build_last_error.restype = C.c_char_p
    rc = L.cfb_synth_reads(C.byref(opts), C.c_uint64(n), C.c_uint32(rdlen), C.c_uint64(seed), _p(out, C.c_uint8))
    if rc != 0:
        raise CfbError("cfb_synth_reads error %d: %s" % (rc, L.cfb_build_last_error().decode()))
    return out


class SynthReadOpts(C.Structure):
    _fields_ = [("len_lo", C.c_uint32), ("len_hi", C.c_uint32), ("paired", C.c_int32), ("ins_lo", C.c_uint32), ("ins_hi", C.c_uint32)]


def synth_reads_ex(opts, n, seed, len_lo, len_hi, paired=False, ins=(200, 500)):
    """-> codes (mates, n, len_hi) uint8 padded with 4, lens (mates, n) uint32"""
    mates = 2 if paired else 1
    ro = SynthReadOpts(len_lo, len_hi, 1 if paired else 0, ins[0], ins[1])
    codes = np.zeros((mates, n, len_hi), dtype=np.uint8); lens = np.zeros((mates, n), dtype=np.uint32)
    L = lib()
    L.cfb_build_last_error.restype = C.c_char_p
    rc = L.cfb_synth_reads_ex(C.byref(opts), C.byref(ro), C.c_uint64(n), C.c_uint64(seed), _p(codes, C.c_uint8), _p(lens, C.c_uint32))
    if rc != 0:
        raise CfbError("cfb_synth_reads_ex error %d: %s" % (rc, L.cfb_build_last_error().decode()))
    return codes, lens


def synth_fasta(opts, path):
    rc = lib().cfb_synth_fasta(C.byref(opts), path.encode())
    if rc != 0:
        raise CfbError("cfb_synth_fasta failed")


def write_synth_taxonomy(outdir, genera, species, length, prefix="seq"):
    """conversion table / nodes.dmp / names.dmp of the synthetic recipe (same as tools/synth.py)."""
    os.makedirs(outdir, exist_ok=True)
    n = genera * species
    with open(os.path.join(outdir, "conv.tsv"), "w") as f:
        for i in range(n):
            f.write("%s%d\t%d\n" % (prefix, i, 1000 + i))
    with open(os.path.join(outdir, "nodes.dmp"), "w") as f:
        f.write("1\t|\t1\t|\tno rank\t|\n")
        for g in range(genera):
            f.write("%d\t|\t1\t|\tgenus\t|\n" % (100 + g))
        for i in range(n):
            f.write("%d\t|\t%d\t|\tspecies\t|\n" % (1000 + i, 100 + i // species))
    with open(os.path.join(outdir, "names.dmp"), "w") as f:
        f.write("1\t|\troot\t|\t\t|\tscientific name\t|\n")
        for g in range(genera):
            f.write("%d\t|\tGenus%d\t|\t\t|\tscientific name\t|\n" % (100 + g, g))
        for i in range(n):
            f.write("%d\t|\tGenus%d species%d\t|\t\t|\tscientific name\t|\n" % (1000 + i, i // species, i))
    return (os.path.join(outdir, "conv.tsv"), os.path.join(outdir, "nodes.dmp"), os.path.join(outdir, "names.dmp"))
