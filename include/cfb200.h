/* include/cfb200.h -- C ABI of the H100-native Centrifuge classification path.
 *
 * This is the batch form of the reference's inner operator boundary: one call
 * classifies a batch of reads/pairs exactly as a sequence of
 *     Classifier::initRead/initReads (hi_aligner.h:739,765) + Classifier::go (classifier.h:212)
 * calls would, against the same `.1-.4.cf` index files that Ebwt<uint64_t> loads
 * (bt2_idx.h:566-854, bt2_io.h:42-685).  The caller is the host worker that replaces
 * multiseedSearchWorker (centrifuge.cpp:2342); it keeps read parsing, the N filter, the
 * per-read RNG / selectByScore tie shuffle (aln_sink.h:1861), TSV formatting and
 * SpeciesMetrics, all of which libcfb200_host provides as well (cfb_run below replaces
 * `extern "C" int centrifuge(int, const char**)`, centrifuge.cpp:3345).
 *
 * Plain C, plain pointers and sizes; nothing throws across this boundary.  All functions
 * return 0 on success or a negative CFB_E* code; cfb_last_error() gives the message.
 * There is no CPU fallback: every classify entry point fails with CFB_ENODEV when no
 * sm_90 (H100) CUDA device is usable.
 */
#ifndef CFB200_H_
#define CFB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CFB_OK        0
#define CFB_EINVAL   -1   /* bad argument */
#define CFB_EIO      -2   /* index / read file problem */
#define CFB_ENOMEM   -3   /* host or device allocation failed */
#define CFB_ENODEV   -4   /* no usable CUDA device (no CPU fallback exists) */
#define CFB_ECUDA    -5   /* CUDA runtime error, see cfb_last_error() */
#define CFB_EFORMAT  -6   /* index geometry not supported by the kernels */
#define CFB_EDATA    -7   /* corrupt or truncated compressed input */

#define CFB_UID_NONE 0xFFFFFFFFu

typedef struct cfb_index cfb_index;   /* immutable, shareable: host arrays + one device replica */
typedef struct cfb_ctx   cfb_ctx;     /* per-thread/per-stream work context; not thread-safe */

/* Replaces: Ebwt<index_t> ctor + loadIntoMemory (centrifuge.cpp:2878,2950).
 * device >= 0 uploads a replica to that GPU; device < 0 loads host tables only
 * (header / taxonomy inspection; classify calls then fail with CFB_ENODEV). */
int cfb_index_load(const char* basename, int device, cfb_index** out);
/* Same, with control over the derived device tables that are built at load time (pure accelerations, results are
 * identical with or without them): the resolve table (sequence id of every SA row, ~0.5 s per Gbp to build) and
 * walk8 (eight LF steps per gather, ~0.25 s per Gbp).  cfb_run skips both for small inputs, where building them
 * would cost more than they save. */
#define CFB_LOAD_NO_RESOLVE_TABLE 1u
#define CFB_LOAD_NO_WALK8         2u
int cfb_index_load_ex(const char* basename, int device, uint32_t flags, cfb_index** out);
void cfb_index_free(cfb_index*);

typedef struct {
	uint64_t len;          /* joined reference length (EbwtParams::_len) */
	uint64_t num_sides;
	uint64_t n_seqs;       /* uid_to_tid().size() */
	uint64_t n_tax_nodes;  /* tree().size() */
	uint64_t n_boundaries; /* .4.cf entries */
	int32_t  line_rate, off_rate, ftab_chars;
	int32_t  sample_bytes; /* 2 or 4 (bt2_io.h:280) */
	int32_t  compressed;   /* Ebwt::compressed(), bt2_idx.h:661 */
	int32_t  device;       /* -1 when host-only */
	uint64_t device_bytes; /* HBM bytes of the replica */
} cfb_index_info;
int cfb_index_get_info(const cfb_index*, cfb_index_info* out);

/* What the device replica holds (bytes of HBM each; 0 = not built).  The derived tables are built at load time in
 * this order of benefit per byte, each only while it fits the budget left after the batch head-room (12 GB unless
 * CFB_HBM_HEADROOM_GB says otherwise; DESIGN.md 3): rank16 + ftab2 (always), the K-mer jump table (whose 16-byte entries
 * also carry the death bitmap), the resolve table, walk8 (possibly for a prefix of the rows).  The file's sides only stage
 * rank16 and are freed once it is built, so sides_bytes is 0 for a rank16 replica.  When rank16 does not fit, the sides are
 * converted in place into the compact rank layout (1/3 byte per row), which sides_bytes then reports with rank16_bytes = 0;
 * such a replica has no resolve table and no walk8 (DESIGN.md 3). */
typedef struct {
	uint64_t sides_bytes, sample_bytes, rank16_bytes, ftab2_bytes, ftabk_bytes, resolve_table_bytes, walk8_bytes;
	uint64_t total_bytes, free_bytes_after_load;
	uint64_t walk8_rows;            /* rows [0, walk8_rows) have a walk8 entry (all rows when HBM allows, else a prefix) */
	uint64_t ftabd_bytes;           /* always 0: the death bitmap (1 bit per (K+3)-mer) lives in the K-mer table's entries */
	int32_t  ftabk_chars;           /* K of the jump table, 0 = none (= ftab_chars when it is built for the death bitmap alone) */
	int32_t  resolve_entry_bytes;   /* 2 or 4, 0 = no resolve table (rows are resolved by walking) */
	int32_t  ftabd_chars;           /* K + 3 while the K-mer table carries the death bitmap, 0 = none */
	int32_t  pad;
} cfb_index_tables;
int cfb_index_get_tables(const cfb_index*, cfb_index_tables* out);

/* Taxonomy accessors the host formatter needs (Ebwt::uid_to_tid/tree/name/size). */
const char* cfb_index_seq_name(const cfb_index*, uint32_t seq);           /* uid string */
uint64_t    cfb_index_seq_taxid(const cfb_index*, uint32_t seq);
/* returns 1 if taxid is a tree node; rank = TaxonomyNode.rank (taxonomy.h:16), leaf flag */
int         cfb_index_tax_node(const cfb_index*, uint64_t taxid, uint64_t* parent, int* rank, int* leaf);
/* all tree taxids in ascending order (n_tax_nodes entries): the index space of dense per-taxon vectors */
int         cfb_index_node_taxids(const cfb_index*, uint64_t* out, uint64_t cap);

/* Replaces: Classifier ctor arguments (classifier.h:135-143) + ReportingParams (aln_sink.h:573). */
typedef struct {
	int32_t khits;            /* -k, default 5 */
	int32_t min_hitlen;       /* --min-hitlen, default 22, clamped to >= 15 (centrifuge.cpp:1401) */
	int32_t tree_traverse;    /* 0 for --no-traverse */
	int32_t class_rank_slot;  /* rank_to_pathID(--classification-rank): 0 strain .. 9 domain; 255 = none */
	const uint64_t* host_taxids;     uint64_t n_host_taxids;      /* --host-taxids as given */
	const uint64_t* excluded_taxids; uint64_t n_excluded_taxids;  /* --exclude-taxids as given */
} cfb_params;
void cfb_params_default(cfb_params*);

/* One context = cfb_ctx_slots() CUDA streams with their device and pinned staging buffers, bound to the index's
 * device.  Buffers are sized by the batches that arrive and grow on demand (about 3.5 KB of HBM per read of a batch in
 * flight).  A context is not thread-safe; create one per host thread that submits work. */
int  cfb_ctx_create(const cfb_index*, const cfb_params*, cfb_ctx** out);
void cfb_ctx_destroy(cfb_ctx*);

/* A batch of units.  Unit i is read i (n_mates==1) or pair i (n_mates==2).
 * bases: 1 byte per base, 0..3 = ACGT, 4 = N (BTDnaString encoding, sstring.h), forward
 * strand as parsed.  mate m of unit i lives at bases[off[m][i] .. off[m][i]+len[m][i]).
 * flags[i]: bit0 = mate 1 passes the caller's filters (N/len/qc, centrifuge.cpp:2550-2596),
 * bit1 = mate 2 passes.  A unit with no passing mate yields zero records ("unclassified").
 * All arrays are caller-owned host memory (pinned memory from cfb_host_alloc is fastest). */
typedef struct {
	uint64_t n_units;
	int32_t  n_mates;            /* 1 or 2 */
	const uint8_t*  bases;  uint64_t n_bases;
	const uint64_t* off[2];
	const uint32_t* len[2];
	const uint8_t*  flags;       /* NULL = all mates pass */
} cfb_batch;
/* Read length.  A mate may hold up to CFB_MAX_MATE_LEN bases (2^31 - 1, so that len1 + len2 and cfb_rec.hitlen stay in 32
 * bits); a longer one makes every classify entry point return CFB_EINVAL.  A unit with a mate longer than CFB_LONG_UNIT_LEN
 * bases (a long unit) is searched in parallel segments by kernels of its own, with device memory sized by its own length
 * (about 100 bytes per base of its mates); its records come back in unit order with the others.  When that memory cannot be
 * had the batch fails with CFB_ENOMEM and cfb_last_error() names the lengths. */
#define CFB_MAX_MATE_LEN  2147483647u
#define CFB_LONG_UNIT_LEN 60000u

/* One AlnRes worth of data (aligner_result.h:321): what Classifier::go hands sink.report(). */
typedef struct {
	uint64_t taxid;
	uint32_t score;
	uint32_t hitlen;    /* (uint64_t)summedHitLen */
	uint32_t uid;       /* sequence index, CFB_UID_NONE after tree traversal merged it */
	uint32_t pad;
} cfb_rec;

/* Library-owned result of one batch; valid until the next submit on the same slot.
 * Records of unit i are recs[rec_off[i] .. rec_off[i+1]), in Classifier::_hitMap order.
 * rec_off[i]==rec_off[i+1] means the reference would have called reportUnclassified(). */
typedef struct {
	uint64_t n_units;
	uint64_t n_recs;
	const uint32_t* rec_off;   /* n_units+1 entries */
	const cfb_rec*  recs;
} cfb_result;

/* Synchronous: H2D, kernels, D2H, returns when the result is in host memory. */
int cfb_classify_batch(cfb_ctx*, const cfb_batch*, cfb_result* out);

/* Pipelined: up to cfb_ctx_slots() batches in flight on independent streams.  Arrays that live in pinned memory
 * (cfb_host_alloc) are DMA'd from where they are and must stay untouched until the matching wait; pageable arrays are
 * copied into pinned staging before submit returns.  The records follow the kernels home without a size round trip,
 * so a wait is normally a single stream synchronisation. */
int cfb_ctx_slots(const cfb_ctx*);
int cfb_classify_submit(cfb_ctx*, int slot, const cfb_batch*);
int cfb_classify_wait(cfb_ctx*, int slot, cfb_result* out);

/* Packed form of a batch: a third of the host->device bytes of the byte form -- about 37 instead of 113 bytes per
 * 100 bp read -- for callers that feed several GPUs from one host.  words: 2 bits per base (A=0 C=1 G=2 T=3), base j of a mate
 * in bits 2*(j&31) of its word j>>5; every mate starts on a word boundary; layout = mate 1 of units 0..n-1, then
 * mate 2 of units 0..n-1, so offsets are implied by the lengths (n_words must equal the sum of ceil(len/32)).
 * n_pos: the positions that hold N instead of the packed code, (word index << 5) | base-in-word.
 * Same results as the byte form (tests/test_gpu_parity.py).  cfb_pack_batch converts a cfb_batch on the host. */
typedef struct {
	uint64_t n_units;
	int32_t  n_mates;
	const uint64_t* words;  uint64_t n_words;
	const uint32_t* len[2];
	const uint64_t* n_pos;  uint64_t n_n;
	const uint8_t*  flags;       /* as in cfb_batch */
} cfb_batch_packed;
int cfb_classify_submit_packed(cfb_ctx*, int slot, const cfb_batch_packed*);     /* collect with cfb_classify_wait */
int cfb_pack_batch(const cfb_batch* in, uint64_t* words, uint64_t words_cap, uint64_t* n_pos, uint64_t npos_cap, uint64_t* n_words, uint64_t* n_n);

/* Device-resident variant used by the roofline measurement: inputs already in HBM
 * (uploaded once by cfb_batch_upload), only kernels run.  kernel_ms (optional, 5 floats)
 * receives CUDA-event times of {search, prep+rows, resolve, score+compact, total}. */
typedef struct cfb_dbatch cfb_dbatch;
int  cfb_batch_upload(cfb_ctx*, const cfb_batch*, cfb_dbatch** out);
void cfb_dbatch_free(cfb_ctx*, cfb_dbatch*);
int  cfb_classify_resident(cfb_ctx*, cfb_dbatch*, float* kernel_ms, uint64_t* n_recs);
/* the same over units [first, first + count) of the uploaded batch (work buffers are sized by the window) */
int  cfb_classify_resident_range(cfb_ctx*, cfb_dbatch*, uint64_t first, uint64_t count, float* kernel_ms, uint64_t* n_recs);
/* copy the last resident result to host (for parity checks) */
int  cfb_resident_result(cfb_ctx*, cfb_result* out);

/* ---- text-level operator (SURVEY.md 8f rank 1): read-file bytes in, classification TSV out -------
 * Replaces, for well-formed input, the per-read host work either side of Classifier::go:
 *   FastqPatternSource/FastaPatternSource::parse + genRandSeed   pat.cpp:725-1157, pat.h:55-91
 *   nFilter / lenfilt                                             centrifuge.cpp:2550-2596
 *   AlnSinkWrap::finishRead -> selectByScore -> AlnSinkSam::append   aln_sink.h:1634-1927,2280-2337
 *   SpeciesMetrics::addSpeciesCounts                              aln_sink.h:142-172
 * `text_a` (`text_b` = mate 2 or NULL) hold exactly `n_records` complete records in the strict layout
 * (FASTQ: 4 lines, FASTA: 2 lines per record, '\n' line ends, last line terminated) and start at a
 * record start.  Tokenising, base conversion, filters, seeds, classification, tie selection and TSV
 * formatting all run on the device; the host only moves bytes.  Anything the strict layout does not
 * cover (CR, blank or wrapped lines, empty names or reads, short quality strings, more hits than the
 * on-device selector holds) sets `irregular` and produces no output: the caller then parses that span
 * with its own reader and uses cfb_classify_submit (cf_host.cpp does exactly that), so results never
 * depend on which path ran. */
typedef struct {
	int32_t  fasta;            /* 0 = FASTQ, 1 = FASTA */
	int32_t  trim5, trim3;
	uint32_t seed;             /* --seed */
	uint32_t maxlen_hint;      /* longest read expected (0 = unknown): sizes the first pass; longer reads only cost a re-run */
} cfb_text_opts;
typedef struct {
	uint64_t n_units;
	int32_t  irregular;        /* != 0: nothing was produced for this span */
	uint32_t maxlen;
	const char* tsv; uint64_t tsv_bytes;        /* rows in input order, pinned host memory */
	/* reads whose best rows tie between several taxa at full score (SpeciesMetrics::observed keys of
	 * size > 1): n_multi records of `multi_stride` u64 = {n, n taxids ascending, ...} */
	const uint64_t* multi; uint64_t n_multi; uint32_t multi_stride;
} cfb_text_result;
int cfb_text_submit(cfb_ctx*, int slot, const void* text_a, uint64_t bytes_a, const void* text_b, uint64_t bytes_b,
                    uint64_t n_records, const cfb_text_opts*);
/* discard != 0: drop the span's contribution to the per-taxon counters (the caller re-does it). */
int cfb_text_wait(cfb_ctx*, int slot, int discard, cfb_text_result* out);
/* Columns of the rows of later cfb_text_submit calls on this context: a `centrifuge-class --tab-fmt-cols` list (comma
 * separated names; readID, seqID, taxID, taxRank/taxLevel, taxName, score, 2ndBestScore, hitLength, queryLength,
 * numMatches, readSeq, readQual, readSeq1/SEQ1, readSeq2/SEQ2, readQual1/QUAL1, readQual2/QUAL2 and the SAM names
 * QNAME, FLAG, RNAME, POS, MAPQ, CIGAR, RNEXT, PNEXT, TLEN, SEQ, QUAL), at most 64 of them.  NULL = the default list
 * readID,seqID,taxID,score,2ndBestScore,hitLength,queryLength,numMatches.  Rows carry no header line.  An unknown name
 * returns CFB_EINVAL with "Column definition <name> invalid." in cfb_last_error(). */
int cfb_ctx_set_columns(cfb_ctx*, const char* cols);
/* N ceiling of later cfb_text_submit calls on this context (`centrifuge-class --n-ceil`): a mate of `len` bases passes
 * the N filter when it holds at most max(min, min(max, constant + coeff * g(len))) bases N or '.', converted to an
 * integer as the reference does, with g = 0, len, sqrt(len) or ln(len) for `type` 1 (constant), 2 (linear), 3 (square
 * root) or 4 (natural log).  The default is type 2, constant 0, coeff 0.15, min 0, max DBL_MAX.  Mates are filtered
 * apart.  A bad type or a NaN parameter returns CFB_EINVAL.  cfb_classify_submit callers pass their own filter flags; the
 * ceiling still sizes the hit lists of their later batches for the Ns a passing mate may hold (a batch whose flags pass
 * more Ns than that is re-run with lists of one entry per base).  A hit list that does not fit returns CFB_ENOMEM.
 * A span or batch keeps the ceiling it was submitted under. */
int cfb_ctx_set_n_ceil(cfb_ctx*, int type, double constant, double coeff, double min, double max);
/* Quality encoding of the FASTQ text of later cfb_text_submit calls (--solexa-quals, --phred64, --int-quals; all 0 is
 * phred33, the default).  Qualities are converted to phred33 for the per-read seed and the quality columns, as the
 * reference does (charToPhred33 / intToPhred33, qual.h:105-171); a span whose qualities the reference would refuse is
 * returned irregular, for the record-level reader to decide.  A span keeps the encoding it was submitted under, re-runs
 * included.  Each argument must be 0 or 1 (else CFB_EINVAL). */
int cfb_ctx_set_quals(cfb_ctx*, int solexa, int phred64, int integer);
/* Per-taxon counters accumulated on the device by all accepted spans: entries with n_reads > 0.
 * n_obs1 = reads whose single best row reached the maximum score (observed keys of size 1). */
int cfb_text_species(cfb_ctx*, uint64_t* taxid, uint64_t* n_reads, uint64_t* n_unique, uint64_t* n_obs1, uint64_t cap, uint64_t* n);

/* ---- per-taxon counters and the multi-GPU reduction (SURVEY.md 8e) ---------------------------------
 * Replaces: SpeciesMetrics::addSpeciesCounts (aln_sink.h:142-172) and, across GPUs, the dense part of
 * SpeciesMetrics::merge (aln_sink.h:109-140; per-thread metrics summed at the end of the run, centrifuge.cpp:3175-3179).
 * Every context keeps, on its device, {numReads, numUniqueReads, reads whose single best row reached the maximum
 * score} for every taxid a report can mention (tree nodes, sequence taxids, 0 = unclassified, 1); the index space is
 * cfb_counts_taxids (ascending).  The text operator always counts; the record-level entry points count when
 * cfb_ctx_count_records is on (a kernel behind the classification kernels of each batch; batches add to the totals when
 * they are waited for).  A unit counts its records of the best score, at most -k of them.  When more than -k records tie
 * for the best score (only under --host-taxids), the text operator picks -k of them with the read's RNG, as the
 * reference does; the record-level counters take the first -k in record (hit-map) order, since cfb_batch carries no
 * per-read seeds.  cfb_counts_allreduce is the path's one collective: ncclAllReduce(ncclUint64, ncclSum) of the
 * totals over the communicator, NVLink/NVSwitch underneath.  The sparse tie sets that feed the EM (cfb_text_result.multi)
 * are merged by the caller, as the reference merges `observed`. */
int cfb_ctx_count_records(cfb_ctx*, int on);
int cfb_counts_taxids(cfb_ctx*, uint64_t* taxid, uint64_t cap, uint64_t* n);
int cfb_counts_reset(cfb_ctx*);
/* entries with n_reads > 0; global = 0: this context's totals, 1: the totals of the last cfb_counts_allreduce */
int cfb_counts_read(cfb_ctx*, int global, uint64_t* taxid, uint64_t* n_reads, uint64_t* n_unique, uint64_t* n_obs1, uint64_t cap, uint64_t* n);
/* dense form: out[0..n) numReads, out[n..2n) numUniqueReads, out[2n..3n) observed singletons, n = cfb_counts_taxids */
int cfb_counts_dense(cfb_ctx*, int global, uint64_t* out, uint64_t cap);
/* Communicator: either one process per GPU (rank 0 calls cfb_comm_unique_id, ships the 128 bytes to the other ranks by
 * whatever launcher plumbing it has, every rank calls cfb_comm_init_rank), or one process driving several GPUs
 * (cfb_comm_init_all over its contexts, one per device; what `centrifuge-class --devices` does). */
#define CFB_COMM_ID_BYTES 128
int cfb_comm_unique_id(uint8_t id[CFB_COMM_ID_BYTES]);
int cfb_comm_init_rank(cfb_ctx*, int nranks, int rank, const uint8_t id[CFB_COMM_ID_BYTES]);
int cfb_comm_init_all(cfb_ctx* const* ctxs, int n);
int cfb_comm_info(const cfb_ctx*, int* rank, int* size, int* nccl_version);
/* ctxs = the calling process's contexts (n = 1 under torchrun/MPI); collective over the communicator.  dense_out
 * (optional) receives the reduced dense vector (layout of cfb_counts_dense).  Without a communicator and n = 1 the
 * "reduced" totals are the local ones. */
int cfb_counts_allreduce(cfb_ctx* const* ctxs, int n, uint64_t* dense_out, uint64_t cap);

/* Measurement hooks (bench.py): the product's own load requests of the last batch when the context was created with
 * CFB_COUNT=2 -- {rank16 entries, 10-mer table entries, K-mer table entries, walk8 entries, 0} -- and the random-gather
 * ceiling of this device over the replica's own arrays: independent uniformly random gathers from table 0 = rank16
 * (16 B), 1 = K-mer table (16 B), 2 = walk8 (8 B), 3 = resolve table (8 B), in G requests/s; 4 (death bits: no table of their own) always fails as not built. */
int cfb_ctx_requests(cfb_ctx*, uint64_t out[5]);
/* Where those requests go (CFB_COUNT=2): {rank16 requests made while the range has width 1, width 2-4, width >= 5 (the three sum
 * to the rank16 entries above), walk8 jumps tried from a single row, taken from a single row, tried from a range, taken from a
 * range, taken from a range of width >= 5}.  A separate call, so that the sum of cfb_ctx_requests stays the total request count. */
int cfb_ctx_request_breakdown(cfb_ctx*, uint64_t out[8]);
int cfb_gather_ceiling(const cfb_index*, int table, uint64_t n_requests, double* g_requests_per_s, double* ms);
/* The same probe with a chosen number of requests in flight: ctas_per_sm CTAs of 128 threads per SM, ilp (1, 2 or 4) independent
 * requests per thread.  cfb_gather_ceiling is (16, 4); the search kernel's own shape is (8, 1). */
int cfb_gather_rate(const cfb_index*, int table, uint64_t n_requests, int ctas_per_sm, int ilp, double* g_requests_per_s, double* ms);
/* How the search kernel's loop spent its trips in the last batch (CFB_COUNT=2): {warp-iterations, lane-iterations that issued a
 * table request, consumer branches with at least one lane summed over warp-iterations, restart blocks (hit store, task hand-out,
 * search start) with at least one lane summed likewise, warp-iterations in which a lane received a task, SM clocks summed over
 * one lane per warp from the loop top to the fetch issue, from there until the loaded data is usable, from there to the end of the trip}. */
int cfb_ctx_search_iter_stats(cfb_ctx*, uint64_t out[8]);
/* How the scoring kernel spent the last batch (CFB_COUNT=1 or 2): {units with rows to score, their rows, their distinct ids,
 * units that entered the tree reduction, rank rounds those ran, warps with rows, warps whose rows did not fit the shared pool},
 * then units by rows and units by distinct ids in eight log2 buckets each (1, 2-3, 4-7, ..., >= 128). */
int cfb_ctx_score_stats(cfb_ctx*, uint64_t out[23]);

/* Operation counters of the last batch on this ctx when it was created with CFB_COUNT=1, which searches with the scalar,
 * table-free restatement of the reference's walk (same definition as SURVEY.md 8d):
 * {units, partial_searches, ftab_probes, sides_search, walk_steps, rows_resolved, lf_steps_total, ext_searches} */
int cfb_ctx_counters(cfb_ctx*, uint64_t out[8]);
/* Long units classified by this ctx so far: {long units, bases of their searched mates, partial searches of the speculative
 * segment chains, partial searches the join ran again}. */
int cfb_ctx_long_stats(const cfb_ctx*, uint64_t out[4]);
int cfb_ctx_kernel_launches(const cfb_ctx*, uint64_t* n);

int   cfb_device_count(void);         /* usable CUDA devices (0 without a driver) */
void* cfb_host_alloc(size_t bytes);   /* pinned host memory (portable: every device of the process can DMA from it) */
void  cfb_host_free(void*);

/* Device unit-test hooks (tests/ only): run the product's LF and resolve walk on rank16 over
 * arrays of rows.  out[i] = LF(rows[i], chars[i]) ; chars[i] > 3 means BWT[rows[i]]. */
int cfb_test_lf(const cfb_index*, const uint64_t* rows, const uint8_t* chars, uint64_t n, uint64_t* out);
int cfb_test_resolve(const cfb_index*, const uint64_t* rows, uint64_t n, uint32_t* out);
/* Host-only test hook: the record-level FASTA/FASTQ reader of cfb_run over a file; one line per read
 * "name<TAB>bases<TAB>seed<TAB>passes filters".  Returns 1 where the reference would stop with an error. */
int cfb_test_parse(const char* path, int fasta, int trim5, int trim3, uint32_t seed, const char* out_path);
/* Host-only test hook: the whole host side of the record-level path (reader, seeds, filters, tie selection, rows,
 * metrics, EM, report, Kraken-style report) around classification records supplied by the caller. */
int cfb_test_host_path(const char* index_base, const char* reads_a, const char* reads_b, int fasta, int khits, uint32_t seed,
                       int trim5, int trim3, const uint32_t* rec_off, const cfb_rec* recs, uint64_t n_units,
                       const char* out_tsv, const char* out_report, const char* out_kreport);

const char* cfb_last_error(void);
const char* cfb_version(void);

/* ---- gzip inflater: RFC 1952 members of RFC 1951 DEFLATE data, decompressed on the device -------------
 * Byte for byte what zlib produces, for every block type, header flag and member layout (several members, empty ones,
 * BGZF).  Each member's CRC-32 and ISIZE are checked.  The compressed stream is cut into chunks of `chunk_kb` KB (0 =
 * CFB_GZ_CHUNK_KB, else 64) that are decoded in parallel from speculated block starts; a wrong guess is decoded again
 * from the previous chunk's end, so the output never depends on the guesses.  Device memory grows with the chunk size
 * (a pass covers 512 chunks), not with the stream.  There is no host inflate. */
typedef struct cfb_gunzip cfb_gunzip;
int  cfb_gunzip_create(int device, uint32_t chunk_kb, cfb_gunzip** out);
void cfb_gunzip_destroy(cfb_gunzip*);
/* Streaming: feed compressed bytes `in` (the unconsumed tail of the previous call first), get up to out_cap decompressed
 * bytes.  *n_consumed bytes of `in` were used; pass the rest again, followed by more of the file.  in_is_last != 0: `in`
 * reaches the end of the file.  A call that returns n_out == 0 and n_consumed == 0 needs more input, or with in_is_last
 * has finished the file.  Corrupt or truncated data (bad header, reserved block type, invalid code, distance before the
 * start of the member, CRC-32 or ISIZE mismatch, trailing bytes that are not a member) returns CFB_EDATA, and so does
 * every later call.  Bytes delivered before an error belong to members or passes that decoded without one. */
int  cfb_gunzip_run(cfb_gunzip*, const void* in, uint64_t n_in, int in_is_last, void* out, uint64_t out_cap,
                    uint64_t* n_out, uint64_t* n_consumed);
/* Resume state between two calls when no output is pending (after a call that filled less than out_cap): restore it
 * into any inflater and feed the file from in_offset to continue with byte out_offset of the decompressed stream. */
typedef struct {
	uint64_t in_offset;        /* compressed bytes consumed before this state */
	uint64_t out_offset;       /* decompressed bytes produced before this state */
	uint64_t bit;              /* next bit to decode, counted from in_offset */
	uint64_t hdr_bit;          /* header of the Huffman block being decoded (~0: at a block boundary), from in_offset */
	uint64_t member_bytes;     /* decompressed bytes of the current member so far */
	uint32_t crc;              /* their CRC-32 */
	uint32_t win_len;          /* valid bytes at the end of window */
	int32_t  phase;            /* 0: before a member header, 1: inside the DEFLATE data, 2: before the trailer */
	uint32_t members;          /* members completed */
	uint8_t  window[32768];    /* the last 32 KB of the member's output */
} cfb_gunzip_state;
int  cfb_gunzip_get_state(const cfb_gunzip*, cfb_gunzip_state* out);
int  cfb_gunzip_set_state(cfb_gunzip*, const cfb_gunzip_state* in);
/* {members completed, compressed bytes consumed, decompressed bytes produced, chunks decoded, chunks re-decoded} */
int  cfb_gunzip_stats(const cfb_gunzip*, uint64_t out[5]);

/* ---- bzip2 decompressor: bzip2 streams (one or several concatenated), decompressed on the device -------------------
 * Byte for byte what `bzip2 -dc` (libbz2 1.0.8) produces, for every level, concatenated and empty streams.  Each block's
 * CRC and each stream's combined CRC are checked.  Each pass scans `pass_kb` KB of compressed input (0 = CFB_BZ2_PASS_KB,
 * else 65536) for block starts and decodes the blocks it finds in parallel.  Device memory grows with the blocks a pass
 * holds, not with the stream: about 4.8 MB per block (BWT column, tt array, segment tables), at most one block per 128 KB
 * of pass and 512 in all, plus the pass's input and a 64 MB staging buffer (and 64 MB of pinned host memory).  A file
 * with 512 or more blocks per pass therefore takes about 2.6 GB of device memory at the default pass size (a 16 MB
 * pass: 128 blocks, about 0.75 GB); a smaller file takes only what its blocks need.  Randomised blocks (obsolete since
 * bzip2 0.9.5) are rejected, and so is a block that pads one code length with more than 40 +1/-1 steps (no encoder
 * writes more than 19).  There is no host decoder.  CFB_ENODEV without a device. */
typedef struct cfb_bunzip2 cfb_bunzip2;
int  cfb_bunzip2_create(int device, uint32_t pass_kb, cfb_bunzip2** out);
void cfb_bunzip2_destroy(cfb_bunzip2*);
/* Streaming, with the contract of cfb_gunzip_run: feed compressed bytes `in` (the unconsumed tail of the previous call
 * first), get up to out_cap decompressed bytes; *n_consumed bytes of `in` were used.  A call that returns n_out == 0 and
 * n_consumed == 0 needs more input, or with in_is_last has finished the file.  Bytes after a complete stream that do not
 * start with "BZh1".."BZh9" are ignored and counted, as `bzip2 -dc` does.  Corrupt or truncated data (bad block header,
 * invalid selector, code or code length, origPtr out of range, a block longer than its level allows, a block or stream
 * CRC mismatch, a randomised block) returns CFB_EDATA, and so does every later call.  Bytes are delivered only from
 * blocks whose CRC has been checked. */
int  cfb_bunzip2_run(cfb_bunzip2*, const void* in, uint64_t n_in, int in_is_last, void* out, uint64_t out_cap,
                     uint64_t* n_out, uint64_t* n_consumed);
/* {streams completed, compressed bytes consumed, decompressed bytes produced, blocks, rejected block starts (block
 * magics inside other data), trailing bytes ignored} */
int  cfb_bunzip2_stats(const cfb_bunzip2*, uint64_t out[6]);

/* ---- index builder (libcfb200): GPU construction of `.1-.4.cf` ----------------------------
 * Replaces: centrifuge-build-bin (centrifuge_build.cpp:472-560 -> Ebwt::initFromVector /
 * buildToDisk, bt2_idx.h:1247-1640,3379-3840) for lineRate 7 indexes.  Either FASTA inputs, or
 * (n_fasta == 0) counter-based synthetic genomes "seq0..seqN-1" of synth_genera x synth_species
 * sequences of synth_len bases generated on the device (cf_synth.h) -- used by bench.py to obtain a
 * p_compressed-scale index without network access. */
typedef struct {
	const char* out_base;
	const char* const* fasta; int32_t n_fasta;
	uint32_t synth_genera, synth_species; uint64_t synth_len, synth_seed; double synth_div;
	const char* conversion_table;   /* --conversion-table */
	const char* taxonomy_tree;      /* --taxonomy-tree (nodes.dmp) */
	const char* name_table;         /* --name-table (names.dmp), may be NULL */
	const char* size_table;         /* --size-table, may be NULL */
	int32_t ftab_chars, off_rate;   /* defaults 10, 4 (centrifuge_build.cpp:93-97) */
	int32_t device, verbose;
	const char* synth_prefix;       /* synthetic sequence names are <prefix><i>; NULL = "seq".  "cid" makes the index a
	                                   "compressed" one for the classifier (>= 10 names starting with cid, bt2_idx.h:648-663) */
} cfb_build_opts;
void cfb_build_opts_default(cfb_build_opts*);
int  cfb_build_index(const cfb_build_opts*);
const char* cfb_build_last_error(void);
/* n reads of rdlen bases (codes 0..4) sampled from the synthetic genomes of `o`: uniform sequence /
 * position / strand, 1% substitutions, 0.1% N, 5% random reads (SURVEY.md 8d recipe). */
int cfb_synth_reads(const cfb_build_opts* o, uint64_t n, uint32_t rdlen, uint64_t read_seed, uint8_t* out_codes);
int cfb_synth_fasta(const cfb_build_opts* o, const char* path);
/* The same recipe with lengths U[len_lo, len_hi] and, when paired, 2 mates per unit from a fragment of U[ins_lo, ins_hi]
 * bases with mate 2 reverse-complemented (SURVEY.md 8d: 2 x 150 PE, insert 200-500; 75-300 bp mixed lengths).
 * out_codes: (mates, n, len_hi) bytes, rows padded with 4; out_lens: (mates, n). */
typedef struct { uint32_t len_lo, len_hi; int32_t paired; uint32_t ins_lo, ins_hi; } cfb_synth_read_opts;
int cfb_synth_reads_ex(const cfb_build_opts* o, const cfb_synth_read_opts* ro, uint64_t n, uint64_t read_seed, uint8_t* out_codes, uint32_t* out_lens);

/* ---- host driver (libcfb200_host): drop-in for `centrifuge-class` ------------------
 * Replaces: extern "C" int centrifuge(int argc, const char** argv) (centrifuge.cpp:3345).
 * Same argv conventions and exit codes for the options it implements; unknown options
 * are rejected with exit code 1 like the reference's getopt table does. */
int cfb_run(int argc, const char** argv);

/* Abundance EM on the device (SURVEY.md 8f rank 3).  Replaces the iteration of SpeciesMetrics::calculateAbundance
 * (aln_sink.h:274-495; EM step :196-272, SQUAREM extrapolation :430-470) on a flattened tie-set table:
 * key k (k < K, in std::map order of `observed`) was seen count[k] times and contributes to the species slots
 * target[key_off[k] .. key_off[k+1]) in the order the reference's loops visit them; len[j] is the genome size of
 * slot j; p[0..n) holds the start vector and receives the result.  Every accumulator is summed in the reference's
 * order without FMA contraction, so the doubles (and the report text) are identical to the CPU iteration.
 * cfb_run uses it for tables with >= 2^18 contributions (CFB_GPU_EM=1/0 forces it on/off). */
int cfb_em_abundance(int device, uint64_t n, uint64_t K, const uint64_t* count, const uint64_t* key_off, const uint32_t* target,
                     const uint64_t* len, double* p, uint64_t* iters, double* last_diff);
const char* cfb_em_last_error(void);
/* The same iteration on the host (what cfb_run uses for small tables). */
int cfb_em_abundance_host(uint64_t n, uint64_t K, const uint64_t* count, const uint64_t* key_off, const uint32_t* target,
                          const uint64_t* len, double* p, uint64_t* iters, double* last_diff);

/* Kraken-style report (SURVEY.md 8f rank 4).  Replaces the `centrifuge-kreport` script (centrifuge-kreport:60-260,
 * default LCA mode; its --show-zeros / --min-score / --min-length options): same bytes from the same classification
 * TSV and index.  cfb_run produces the same report in-process with `--kreport-file F` (plus --kreport-show-zeros,
 * --kreport-min-score N, --kreport-min-length N) from the rows while they are still in memory.  Host only. */
int cfb_kreport(const char* index_base, const char* tsv_path, const char* out_path, int show_zeros,
                int has_min_score, long long min_score, int has_min_length, long long min_length);

/* Promote the taxIDs of a classification TSV to a taxonomic level, or merge every read's rows into their lowest common
 * ancestor with level "lca" (SURVEY.md 8f rank 4).  Replaces the `centrifuge-promote` script (centrifuge-promote:1-175):
 * same bytes from the same TSV and index; tsv_path / out_path "-" = stdin / stdout.  Host only.  The drop-in binary
 * runs it as `centrifuge-class --promote <index> <tsv> <level>`. */
int cfb_promote(const char* index_base, const char* tsv_path, const char* level, const char* out_path);

#ifdef __cplusplus
}
#endif
#endif /* CFB200_H_ */
