// cf_logic.h -- per-read classification logic shared by the CUDA kernels (device) and the
// CPU unit tests (host compilation, tests/ only; the product never runs this on the host).
//
// Everything here is scalar, branchy, integer code: the parts of Classifier::go that are not
// the bandwidth-bound FM walks, which live in cfb200.cu.
// Reference behaviour restated (paths relative to the reference tree):
//   partialSearch            hi_aligner.h:903-1031
//   searchForwardAndReverse  classifier.h:646-896 (extend / twin removal / trim parts)
//   getForwardOrReverseHit   classifier.h:898-941
//   compareBWTHits + sort    classifier.h:267,1058-1086, ds.h:775-778 (std::sort, libstdc++)
//   go(): resolve loop, hit map, finalize, host rule, tree reduction, emit  classifier.h:212-571
#ifndef CF_LOGIC_H_
#define CF_LOGIC_H_

#include <stdint.h>

#ifdef __CUDACC__
#define CFB_HD __host__ __device__ __forceinline__
#define CFB_HDN __host__ __device__
#else
#define CFB_HD inline
#define CFB_HDN inline
#endif

namespace cfb {

static const uint64_t kOff = 0xffffffffffffffffull;
static const uint64_t kUnk = 0xfffffffffffffffeull;   // HitRec.top == bot == kUnk: a hit shorter than min_hitlen whose SA range was not computed (death bitmap of the K-mer table)
static const uint32_t kBwNone = 0xffffffffu;       // BWTHit::reset(): _bwoff = OFF_MASK

// ----------------------------------------------------------------------------------------
// Device/host view of the index.  Only lineRate 7 (128-byte sides: 96 B of 2-bit BWT = 384
// bases, then occ[A,C,G,T] as 4 x u64 counted before the side) is supported by the kernels.
// ----------------------------------------------------------------------------------------
// What scoring needs of one sequence id under a context's parameters, in one aligned 16-byte record (see seq_info_of).
struct alignas(16) SeqInfo {
	uint64_t taxid;       // after the class_rank_slot resolution
	int32_t  pid;         // path id or -1 (empty path)
	uint32_t flags;       // kSeqExcluded | rank the resolution stopped at << 8
};
static const uint32_t kSeqExcluded = 1u;

struct IndexView {
	const uint64_t* sides;     // num_sides * 16 u64: the host twin's; the device replica frees them once rank16 is built (null)
	const uint64_t* ftab;
	const uint64_t* eftab;
	const uint16_t* sample16;   // exactly one of sample16/sample32 is non-null
	const uint32_t* sample32;
	const uint64_t* brow;       // sorted boundary rows
	const uint32_t* bseq;
	const uint32_t* bbits;      // prefilter bitmap over row >> bshift
	const uint64_t* seq_taxid;
	const int32_t*  seq_path;
	const uint64_t* paths;      // n_paths * 10
	const uint8_t*  seq_excluded;   // per-sequence flag (host views only: the device reads it through `seqs`; may be null)
	const uint64_t* host_taxids;    // sorted expanded host set (per ctx)
	const SeqInfo*  seqs;           // per ctx: seq_info_of every sequence id (null: computed from the arrays above)
	const uint64_t* rank16;         // device-only rank entries: 16 bytes (occ_c, 64 indicator bits) per (64 rows, base); format and decoders below
	const uint64_t* ftab2;          // device-only fused ftab: (top, bot) per 10-mer, eftab already resolved
	const uint16_t* rtab16;         // device-only resolve table: sequence id of EVERY SA row (one of rtab16/rtab32, or neither)
	const uint32_t* rtab32;
	const uint64_t* ftabk;          // device-only K-mer jump table: (top | width << 40, death bitmap) per K-mer, K = ftabk_chars, see k_build_ftabk (null = absent)
	const uint64_t* cr;             // device-only compact rank layout (when rank16 does not fit): 64-byte half-sides, format and decoders below (null = absent)
	const uint64_t* crsb;           // its superblock table: occ of every base before each superblock's first half-side, 4 x u64 per superblock
	const uint64_t* walk8;          // device-only: per SA row, the row 8 LF steps on | the 8 BWT bases met << 40 | #valid steps << 56 (null = absent)
	uint64_t walk8_rows;            // rows [0, walk8_rows) have a walk8 entry (the table may cover a prefix of the rows when HBM is short)
	int32_t  ftabd_chars;           // K + 3 while the K-mer table carries the death bitmap, else 0
	uint64_t len, zoff, zside, fchr[4], last_boundary, num_sides;
	uint32_t zoffc, n_boundaries, n_seqs, n_host;
	int32_t  off_rate, ftab_chars, bshift, ftabk_chars;
};

struct Params {
	uint32_t khits, min_hitlen, ihits, increment;
	uint32_t tree_traverse, class_rank_slot;
};

struct HitRec { uint64_t top, bot; uint32_t bwoff, len; };   // 24 bytes

// A row queued for resolution carries the plan of the scoring pass in its high bits, so that pass reads one
// contiguous array instead of gathering the hit lists again: the first row of every counted hit has kRowStart set
// plus the hit length (bits 40..55), the list it came from (mate bit 56, strand bit 57) and kRowSameTs when the hit
// carries the same time stamp as the previous counted hit.  That happens in the reference when a list loop is left
// through its `break` (the loop-header ts++ is skipped, classifier.h:283-345) and the next list starts with a counted
// hit: the second hit then does not add its score to entries the first one touched -- a quirk the output depends on.
// SA rows need 40 bits.
static const uint64_t kRowMask = (1ull << 40) - 1ull, kRowStart = 1ull << 63, kRowSameTs = 1ull << 58;

struct Counters {   // algorithmic-operation counters (SURVEY.md section 8d definition)
	unsigned long long units, partial_searches, ftab_probes, sides_search, walk_steps, rows_resolved, lf_steps, ext_searches;
	// the product's own load requests (count mode 2: every derived table live, one entry per lane-level gather):
	// rank16 entries (16 B), 10-mer table entries (16 B), K-mer table entries (16 B), walk8 entries (8 B); req_ftabd stays 0
	// (the death bitmap is read with the K-mer table entry)
	unsigned long long req_rank16, req_ftab2, req_ftabk, req_walk8, req_ftabd;
	// where the requests of count mode 2 go: rank16 requests made while the range has width 1, 2-4 and >= 5 (they sum to
	// req_rank16), and walk8 jumps tried and taken from a single row and from a range (w8_ok_w5: taken from width >= 5)
	unsigned long long r16_w1, r16_w2_4, r16_w5, w8_try_row, w8_ok_row, w8_try_range, w8_ok_range, w8_ok_w5;
	// how k_search_t's loop spends a trip (count mode 2): warp-iterations, lane-iterations that issued a table request,
	// distinct consumer branches and distinct restart blocks (hit store, hand-out, search start) with at least one lane,
	// summed over warp-iterations, warp-iterations in which a lane received a task, and SM clocks summed by lane 0 over
	// loop top -> fetch issue, fetch issue -> loaded data usable, loaded data usable -> end of the trip
	unsigned long long it_warp, it_lane_req, it_consumers, it_restarts, it_task, clk_head, clk_wait, clk_tail;
	// how k_score spends a batch (count modes 1 and 2): units with rows to score, their rows, their distinct ids (hit-map
	// entries), units that enter the tree reduction and the rank rounds they run, warps with rows and warps whose rows did not
	// fit the shared pool (global scratch); rows and distinct ids per unit in log2 buckets (0: 1, 1: 2-3, ..., 7: >= 128)
	unsigned long long sc_units, sc_rows, sc_nmap, sc_reduce, sc_rounds, sc_warps, sc_warps_global;
	unsigned long long sc_rows_hist[8], sc_nmap_hist[8];
};

CFB_HD int popc64(uint64_t x) {
#ifdef __CUDA_ARCH__
	return __popcll(x);
#else
	return __builtin_popcountll(x);
#endif
}
CFB_HD uint32_t ctz32(uint32_t x) {      // x != 0
#ifdef __CUDA_ARCH__
	return (uint32_t)(__ffs(x) - 1);
#else
	return (uint32_t)__builtin_ctz(x);
#endif
}

// rank16 (IndexView::rank16): for every 64 rows and every base c one 16-byte entry
//   u64 occ_c (count of c before the block, '$' excluded; bit 63 of A's entry = "block holds a genome-boundary row")  |
//   u64 indicator bits (BWT[row] == c; the '$' row has no bit)
// so LF(row, c) = fchr[c] + occ + popc(bits & lowmask(row & 63)).  Every kernel addresses and decodes entries through these two.
static const uint64_t kOccMask = 0x7fffffffffffffffull;
// index of the entry of (row, c) in 16-byte units; the four bases of a block share one 64-byte chunk
CFB_HD uint64_t r16_entry(uint64_t row, int c) { return (row >> 6) * 4 + (uint64_t)c; }
// LF(row, c) from the entry of (row, c)
CFB_HD uint64_t r16_lf(const IndexView& v, uint64_t row, int c, uint64_t occ, uint64_t bits) {
	return v.fchr[c] + (occ & kOccMask) + (uint64_t)popc64(bits & (((uint64_t)1 << (row & 63)) - 1));
}

// walk8 (k_build_walk8): per SA row r, the row eight successive mapLF1 steps reach (bits 0-39), the eight BWT bases met on the
// way (2 bits each from bit 40, first step lowest) and the number of valid steps (bits 56-63; fewer than 8 when the walk meets
// the '$' row).  walk8_steps = how many of the next eight read bases (`win`: 2 bits each, base p in bits 2p; N bits in `nwin`)
// row r follows: 8 = all of them, else the step at which it leaves the range (a different base, an N, or the '$' row).
//
// Range rule.  The range of cP is the set of LF images of the rows of P's range [top, bot) whose BWT base is c; LF keeps
// their order, so when top and bot - 1 both have base c the new range is exactly [LF(top), LF(bot - 1) + 1), whatever the
// rows between them do.  By induction: when both end rows follow all eight bases, the range after them is exactly
// [W8(top), W8(bot - 1) + 1) -- possibly narrower (interior rows may drop out), never empty.  And an end row stays the end
// of the range for as long as it follows the read, so after a failed attempt every jump tried before both failing ends have
// left fails the same way: walk8_retry is the first step from which the next attempt can succeed.
static const uint64_t kWalkRowMask = (1ull << 40) - 1ull;
CFB_HD uint32_t walk8_steps(uint64_t e, uint64_t win, uint32_t nwin) {
	const uint32_t diff = (uint32_t)(((e >> 40) ^ win) & 0xffffull), nb = nwin & 0xffu, nv = (uint32_t)(e >> 56);
	uint32_t good = diff ? ctz32(diff) >> 1 : 8u;
	if(nb) { const uint32_t n = ctz32(nb); good = n < good ? n : good; }
	return nv < good ? nv : good;
}
CFB_HD uint32_t walk8_retry(uint32_t st, uint32_t sb) {     // steps of the two end rows, at least one below 8
	const uint32_t a = st < 8u ? st : 0u, b = sb < 8u ? sb : 0u;
	return (a > b ? a : b) + 1u;
}

// positions (bit 2i) where the 2-bit code at i equals c
CFB_HD uint64_t match2(uint64_t w, int c) {
	uint64_t y = ~(w ^ ((uint64_t)c * 0x5555555555555555ull));
	return y & (y >> 1) & 0x5555555555555555ull;
}

// Compact rank layout (IndexView::cr, 1/3 byte per row): half-side h covers rows [192h, 192h + 192) in 64 bytes:
//   u32 cnt[4] (occ of c before the half-side, '$' excluded, minus the superblock's entry)  |  6 x u64 of 2-bit BWT, 32 rows each
// The '$' row is stored as A and corrected for (the zOff rule of countBt2Side, bt2_idx.h:2192-2227); padding after the last row
// reads as A.  Side i of the .1.cf file becomes half-sides 2i and 2i+1 in the same 128 bytes (cr_convert_side), so the layout is
// built in place from the streamed sides.  A superblock is 2^SB half-sides; crsb holds the absolute occ before its first
// half-side.  A rank query reads the count piece and the words before its offset: one 32-byte sector for offsets up to 64, two
// beyond.  SB >= 1 (a superblock starts on a side) and 192 << SB < 2^32 (the relative counts fit their 32 bits).
static const uint32_t kCrRows = 192;
static const int kCrSbShift = 24;           // 2^24 half-sides = 3.2 G rows per superblock
template <int SB> struct CrSbCheck { static_assert(SB >= 1 && (192ull << SB) < (1ull << 32), "superblock span out of range"); };
// number of half-sides including the sentinel one past the last side (an exclusive bound len + 1 on a side boundary reads it)
CFB_HD uint64_t cr_halves(uint64_t num_sides) { return 2 * num_sides + 1; }
template <int SB = kCrSbShift> CFB_HD uint64_t cr_superblocks(uint64_t num_sides) { return (cr_halves(num_sides) + (1ull << SB) - 1) >> SB; }
// occ of c in the 2-bit words w[0, nw) ('$' at position zpos counted out when zpos < 32 * nw)
CFB_HD void cr_count_words(const uint64_t* w, int nw, uint64_t zpos, uint64_t occ[4]) {
	for(int k = 0; k < nw; k++) for(int c = 0; c < 4; c++) occ[c] += (uint64_t)popc64(match2(w[k], c));
	if(zpos < (uint64_t)nw * 32) occ[0] -= 1;
}
// crsb entry of superblock sb, read from the file's sides before they are converted
template <int SB = kCrSbShift> CFB_HD void cr_sb_entry(const uint64_t* sides, uint64_t num_sides, uint64_t zoff, uint64_t sb, uint64_t* out) {
	(void)CrSbCheck<SB>();
	const uint64_t s = sb << (SB - 1);
	if(s < num_sides) { for(int c = 0; c < 4; c++) out[c] = sides[s * 16 + 12 + c]; return; }
	const uint64_t* w = sides + (num_sides - 1) * 16;        // the sentinel half-side's superblock: the totals
	uint64_t occ[4] = {w[12], w[13], w[14], w[15]};
	cr_count_words(w, 12, zoff - (num_sides - 1) * 384, occ);
	for(int c = 0; c < 4; c++) out[c] = occ[c];
}
// Side i -> half-sides 2i, 2i+1 in place (the last side also writes the sentinel half-side into the 64 bytes after it).  Reads
// the whole side before it writes, so one thread per side needs no second copy.  sb: the finished superblock table.
template <int SB = kCrSbShift> CFB_HD void cr_convert_side(uint64_t* sides, uint64_t num_sides, uint64_t zoff, const uint64_t* sb, uint64_t i) {
	(void)CrSbCheck<SB>();
	uint64_t w[16];
	for(int k = 0; k < 16; k++) w[k] = sides[i * 16 + k];
	uint64_t occ[4] = {w[12], w[13], w[14], w[15]};
	const uint64_t zpos = zoff - i * 384;      // wraps to a huge value when '$' lies before the side
	uint64_t* out = sides + i * 16;
	const int nh = i + 1 == num_sides ? 3 : 2;
	for(int k = 0; k < nh; k++) {
		const uint64_t h = 2 * i + (uint64_t)k, base = (h >> SB) * 4;
		out[k * 8] = (occ[0] - sb[base]) | ((occ[1] - sb[base + 1]) << 32);
		out[k * 8 + 1] = (occ[2] - sb[base + 2]) | ((occ[3] - sb[base + 3]) << 32);
		for(int j = 0; j < 6; j++) out[k * 8 + 2 + j] = k < 2 ? w[k * 6 + j] : 0ull;
		if(k < 2) cr_count_words(w + k * 6, 6, zpos - (uint64_t)k * 192, occ);
	}
}
// LF(row, c) and BWT[row] on the compact layout.  The device reads the second sector only when the offset needs it.
template <int SB = kCrSbShift> CFB_HD uint64_t cr_lf(const IndexView& v, uint64_t row, int c) {
	const uint64_t h = row / kCrRows; const uint32_t o = (uint32_t)(row - h * kCrRows);
	const uint64_t* p = v.cr + h * 8;
	uint64_t q[8];
#ifdef __CUDA_ARCH__
	const ulonglong2 a = __ldg(reinterpret_cast<const ulonglong2*>(p)), b = __ldg(reinterpret_cast<const ulonglong2*>(p) + 1);
	q[0] = a.x; q[1] = a.y; q[2] = b.x; q[3] = b.y; q[4] = q[5] = q[6] = q[7] = 0;
	if(o > 64) {
		const ulonglong2 d = __ldg(reinterpret_cast<const ulonglong2*>(p) + 2), e = __ldg(reinterpret_cast<const ulonglong2*>(p) + 3);
		q[4] = d.x; q[5] = d.y; q[6] = e.x; q[7] = e.y;
	}
#else
	for(int k = 0; k < 8; k++) q[k] = p[k];
#endif
	const uint32_t full = o >> 5, rem = o & 31;
	uint64_t n = ((c < 2 ? q[0] : q[1]) >> (32 * (c & 1))) & 0xffffffffull;
#ifdef __CUDA_ARCH__
	#pragma unroll
#endif
	for(uint32_t k = 0; k < 6; k++) {
		const uint64_t m = k < full ? ~0ull : (k == full ? (((uint64_t)1 << (2 * rem)) - 1) : 0ull);
		n += (uint64_t)popc64(match2(q[2 + k], c) & m);
	}
	if(c == 0 && v.zoff < row && v.zoff >= row - o) n--;
	return v.fchr[c] + v.crsb[(h >> SB) * 4 + (uint64_t)c] + n;
}
CFB_HD int cr_bwt(const IndexView& v, uint64_t row) {
	const uint64_t h = row / kCrRows; const uint32_t o = (uint32_t)(row - h * kCrRows);
	return (int)((v.cr[h * 8 + 2 + (o >> 5)] >> ((o & 31) * 2)) & 3);
}

// Which rank layout a replica loads (cfb_index_load_ex), decided from free device memory before anything is allocated:
// rank16 when the transient sides, rank16, the sample, the fixed tables and the head-room all fit; else the compact layout when
// it, the sample, the fixed tables and the head-room fit; else none (-1).  force_compact skips rank16.
enum { kLayoutNone = -1, kLayoutRank16 = 0, kLayoutCompact = 1 };
CFB_HD uint64_t rank16_bytes_for(uint64_t num_sides) { return (num_sides * 6 + 1) * 64; }
CFB_HD uint64_t cr_bytes_for(uint64_t num_sides) { return num_sides * 128 + 64; }
inline int choose_rank_layout(uint64_t free_b, uint64_t num_sides, uint64_t sample_b, uint64_t fixed_b, uint64_t headroom, bool force_compact) {
	const uint64_t rest = sample_b + fixed_b + headroom;
	if(!force_compact && num_sides * 128 + rank16_bytes_for(num_sides) + rest <= free_b) return kLayoutRank16;
	if(cr_bytes_for(num_sides) + rest <= free_b) return kLayoutCompact;
	return kLayoutNone;
}

CFB_HD int bwt_char(const IndexView& v, uint64_t row) {
#ifdef __CUDA_ARCH__
	if(v.rank16) {     // device replica: the indicator bits of the row's 64-row block (one 64-byte chunk); the '$' row has no bit and reads as A, as the file stores it
		const uint32_t o = (uint32_t)(row & 63);
		auto bit = [&](int c) -> uint64_t { return (v.rank16[r16_entry(row, c) * 2 + 1] >> o) & 1ull; };
		return (int)(bit(1) * 1 + bit(2) * 2 + bit(3) * 3);
	}
#endif
	if(v.cr) return cr_bwt(v, row);
	uint64_t s = row / 384; uint32_t off = (uint32_t)(row - s * 384);
	return (int)((v.sides[s * 16 + (off >> 5)] >> ((off & 31) * 2)) & 3);
}

// LF(row, c) = fchr[c] + occ_side[c] + rank_c(side, off) - ['$' stored as A lies before off]
// (countBt2Side bt2_idx.h:2192-2227, countUpTo :2364-2425).  Scalar version: one thread reads
// the words it needs.
CFB_HD uint64_t lf_scalar(const IndexView& v, uint64_t row, int c) {
#ifdef __CUDA_ARCH__
	if(v.rank16) {     // device replica: one 16-byte rank16 entry (occ before the block, '$' excluded | indicator bits), same value as below
		const uint64_t* e = v.rank16 + r16_entry(row, c) * 2;
		return r16_lf(v, row, c, e[0], e[1]);
	}
#endif
	if(v.cr) return cr_lf(v, row, c);
	uint64_t s = row / 384; uint32_t off = (uint32_t)(row - s * 384);
	const uint64_t* w = v.sides + s * 16;
	uint32_t full = off >> 5, rem = off & 31;
	uint64_t n = 0;
	for(uint32_t k = 0; k < full; k++) n += (uint64_t)popc64(match2(w[k], c));
	if(rem) n += (uint64_t)popc64(match2(w[full], c) & (((uint64_t)1 << (2 * rem)) - 1));
	if(c == 0 && s == v.zside && v.zoffc < off) n--;
	return v.fchr[c] + w[12 + c] + n;
}

// strand sequence access without materialising the reverse complement:
// strand 0: seq[j] = fw[j]; strand 1: seq[j] = comp(fw[len-1-j])  (Read::constructRevComps)
CFB_HD int seq_at(const uint8_t* fw, uint32_t len, int strand, uint32_t j) {
	if(strand == 0) return fw[j];
	int c = fw[len - 1 - j];
	return c > 3 ? 4 : 3 - c;
}

CFB_HD uint64_t ftab_hi(const IndexView& v, uint64_t e) { return e <= v.len ? e : v.eftab[(e ^ kOff) * 2 + 1]; }
CFB_HD uint64_t ftab_lo(const IndexView& v, uint64_t e) { return e <= v.len ? e : v.eftab[(e ^ kOff) * 2]; }

// One partialSearch from offset `cur` (scalar; used by the rare extend step and by CPU tests).
// Returns the hit it would append and the new cur / done flags.
CFB_HDN void partial_search_scalar(const IndexView& v, const uint8_t* fw, uint32_t len, int strand,
                                   uint32_t cur, HitRec& out, uint32_t& new_cur, bool& done, Counters* ctr) {
	const uint32_t fc = (uint32_t)v.ftab_chars;
	uint32_t offset = cur, dep = cur;
	done = false;
	if(ctr) ctr->partial_searches++;
	if(len - dep < fc) {
		new_cur = len; out.top = out.bot = kOff; out.bwoff = offset; out.len = len - offset; done = true; return;
	}
	for(uint32_t i = 0; i < fc; i++) {
		if(seq_at(fw, len, strand, len - dep - 1 - i) > 3) {
			new_cur = cur + i + 1; out.top = out.bot = kOff; out.bwoff = offset; out.len = new_cur - offset;
			done = new_cur >= len; return;
		}
	}
	uint64_t fi = 0;
	for(uint32_t i = 0; i < fc; i++) fi = (fi << 2) | (uint64_t)seq_at(fw, len, strand, len - dep - fc + i);
	uint64_t top = ftab_hi(v, v.ftab[fi]), bot = ftab_lo(v, v.ftab[fi + 1]);
	if(ctr) ctr->ftab_probes++;
	dep += fc;
	if(bot <= top) {
		new_cur = dep; out.top = out.bot = kOff; out.bwoff = offset; out.len = dep - offset; done = dep >= len; return;
	}
	while(dep < len) {
		int c = seq_at(fw, len, strand, len - dep - 1);
		if(c > 3) break;
		uint64_t t, b;
		if(bot - top != 1) {
			t = lf_scalar(v, top, c); b = lf_scalar(v, bot, c);
			if(ctr) { ctr->lf_steps += 2; ctr->sides_search += ((top % 384) + (bot - top) < 384) ? 1 : 2; }
		} else {
			if(ctr) { ctr->lf_steps += 1; ctr->sides_search += 1; }
			if(bwt_char(v, top) != c || top == v.zoff) break;
			t = lf_scalar(v, top, c); b = t + 1;
		}
		if(b <= t) break;
		top = t; bot = b; dep++;
	}
	out.top = top; out.bot = bot; out.bwoff = offset; out.len = dep - offset;
	new_cur = dep; done = dep >= len;
}

// Whole greedy search of one strand, one LF step at a time.  Used on the host by tests to cross-check kernel output stage
// by stage, and by k_search_long when it counts the reference's operations.
CFB_HDN uint32_t search_strand_scalar(const IndexView& v, const Params& p, const uint8_t* fw, uint32_t len, int strand,
                                      HitRec* hits, uint32_t cap, Counters* ctr) {
	uint32_t cur = 0, n = 0;
	if(len == 0) return 0;
	for(;;) {
		HitRec h; uint32_t nc; bool done;
		partial_search_scalar(v, fw, len, strand, cur, h, nc, done, ctr);
		if(n < cap) hits[n] = h;
		n++;
		cur = nc;
		if(done) break;
		if(h.len > p.increment) cur += 1;
		if(cur + p.min_hitlen >= len) break;
	}
	return n;
}

// ----------------------------------------------------------------------------------------
// Segmented chains (units with a mate longer than kLongUnitLen bases).  Where the greedy chain of search_strand_scalar goes
// after a partial search depends on the position it started at alone (chain_next), so two chains that visit one position
// agree from there on.  A long strand is cut into segments of `seg` bases; a speculative chain starts at each segment's first
// base and runs until it reaches a position at or past the next segment's start (seg_chain).  The join then follows the true
// chain from position 0 (seg_join): wherever it stands on a position the speculative chain of that segment visited, that
// chain's hits are the true ones up to its exit; elsewhere it runs the partial searches itself.  Every hit records the
// position its partial search started at (bwoff), so the visited positions of a segment are its hits' bwoffs, ascending.
// `step(cur, hit, new_cur, done)` is one partial search: partial_search_scalar on the host, the table walk on the device.
// ----------------------------------------------------------------------------------------
static const uint32_t kLongUnitLen = 60000;          // units with a longer mate take the segmented path
static const uint32_t kMaxMateLen = 0x7fffffffu;     // 2^31 - 1: len1 + len2 and a record's summed hit length stay in 32 bits
static const uint32_t kChainEnd = 0xffffffffu;       // seg_chain's exit when the chain ended inside the segment

// the chain's next start after the hit `h` of the partial search from cur (new_cur, done as it returned); false: the chain ends
CFB_HD bool chain_next(const Params& p, uint32_t len, const HitRec& h, uint32_t new_cur, bool done, uint32_t& cur) {
	cur = new_cur;
	if(done) return false;
	if(h.len > p.increment) cur += 1;
	return cur + p.min_hitlen < len;
}

// The speculative chain from `start`: stores one hit per position it visits below `stop` (at most stop - start hits) and
// returns their number; *exit receives the first position >= stop it reached, or kChainEnd.
template <class Step> CFB_HDN uint32_t seg_chain(const Params& p, uint32_t len, uint32_t start, uint32_t stop, Step& step,
                                                 HitRec* hits, uint32_t* exit) {
	uint32_t cur = start, n = 0;
	for(;;) {
		if(cur >= stop) { *exit = cur; return n; }
		HitRec h; uint32_t nc; bool done;
		step(cur, h, nc, done);
		hits[n++] = h;
		if(!chain_next(p, len, h, nc, done, cur)) { *exit = kChainEnd; return n; }
	}
}

// The true chain of the strand, from the speculative chains of its segments: segment k's hits at shits + k * seg (sn[k] of
// them, exit sexit[k]).  Writes the hits search_strand_scalar would produce to out (capacity len) and returns their number;
// *researched counts the partial searches the join ran itself.
template <class Step> CFB_HDN uint32_t seg_join(const Params& p, uint32_t len, uint32_t seg, const HitRec* shits, const uint32_t* sn,
                                                const uint32_t* sexit, Step& step, HitRec* out, unsigned long long* researched) {
	if(len == 0) return 0;
	uint32_t q = 0, n = 0;
	for(;;) {
		const uint32_t k = q / seg, m = sn[k];
		const HitRec* H = shits + (uint64_t)k * seg;
		uint32_t lo = 0, hi = m;
		while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(H[mid].bwoff < q) lo = mid + 1; else hi = mid; }
		if(lo < m && H[lo].bwoff == q) {        // the speculative chain stands here too: it is the true chain up to its exit
			for(uint32_t i = lo; i < m; i++) out[n++] = H[i];
			if(sexit[k] == kChainEnd) return n;
			q = sexit[k];
		} else {
			HitRec h; uint32_t nc; bool done;
			step(q, h, nc, done);
			*researched += 1;
			out[n++] = h;
			if(!chain_next(p, len, h, nc, done, q)) return n;
		}
	}
}

CFB_HD uint64_t bw64(const HitRec& h) { return h.bwoff == kBwNone ? kOff : (uint64_t)h.bwoff; }
CFB_HD uint64_t hsize(const HitRec& h) { return h.bot - h.top; }

// Trimming of overlapping hits within each strand list (the last part of post_search).
CFB_HD void trim_lists(HitRec* F, uint32_t nF, HitRec* R, uint32_t nR) {
	for(int s = 0; s < 2; s++) {
		HitRec* L = s == 0 ? F : R; const uint32_t n = s == 0 ? nF : nR;
		if(n < 2) continue;
		for(uint32_t i = 0; i + 1 < n; i++) {
			for(uint32_t j = i + 1; j < n; j++) {
				const uint64_t abw = bw64(L[i]), bbw = bw64(L[j]);
				if(abw >= bbw) { L[i].len = 0; break; }
				if(abw + L[i].len <= bbw) break;
				if(L[i].len >= L[j].len) {
					const uint64_t e = bbw + L[j].len, nb = abw + L[i].len;
					L[j].bwoff = (uint32_t)nb; L[j].len = (uint32_t)(e - nb);
				} else L[i].len = (uint32_t)(bbw - abw);
			}
		}
	}
}

// Post-search part of searchForwardAndReverse for one mate: extend, twin removal, trim.
CFB_HDN void post_search(const IndexView& v, const Params& p, const uint8_t* fw, uint32_t rdlen,
                         HitRec* F, uint32_t nF, HitRec* R, uint32_t nR, Counters* ctr) {
	const uint64_t minHitLen = p.min_hitlen;
	uint64_t sum[2] = {0, 0};
	for(uint32_t i = 0; i < nF; i++) if(F[i].len >= minHitLen) sum[0] += F[i].len;
	for(uint32_t i = 0; i < nR; i++) if(R[i].len >= minHitLen) sum[1] += R[i].len;
	if(sum[0] >= minHitLen && sum[1] >= minHitLen) {
		for(uint32_t i = 0; i < nF; i++) {
			const uint64_t len = F[i].len, l = bw64(F[i]), r = l + len;     // locals are not refreshed (classifier.h:795-798)
			for(uint32_t j = 0; j < nR; j++) {
				const uint64_t rclen = R[j].len;
				if(len < minHitLen && rclen < minHitLen) continue;
				const uint64_t rc_l = (uint64_t)rdlen - bw64(R[j]) - R[j].len, rc_r = rc_l + rclen;
				if(r <= rc_l) continue;
				if(rc_r <= l) continue;
				if(l == rc_l && r == rc_r) continue;
				if(l < rc_l && r > rc_r) continue;
				if(l > rc_l && r < rc_r) continue;
				if(l > rc_l) {
					HitRec t; uint32_t nc; bool dn;
					if(ctr) ctr->ext_searches++;
					partial_search_scalar(v, fw, rdlen, 0, (uint32_t)rc_l, t, nc, dn, ctr);
					if((uint64_t)t.len == len + l - rc_l) F[i] = t;
				}
				if(r > rc_r) {
					HitRec t; uint32_t nc; bool dn;
					if(ctr) ctr->ext_searches++;
					partial_search_scalar(v, fw, rdlen, 1, (uint32_t)((uint64_t)rdlen - r), t, nc, dn, ctr);
					if((uint64_t)t.len == rclen + r - rc_r) R[j] = t;
				}
			}
		}
		for(uint32_t i = 0; i < nF; i++) {
			const uint64_t len = F[i].len, l = bw64(F[i]), r = l + len;
			for(uint32_t j = 0; j < nR; j++) {
				const uint64_t rclen = R[j].len;
				const uint64_t rc_l = (uint64_t)rdlen - bw64(R[j]) - R[j].len, rc_r = rc_l + rclen;
				if(rc_l < l) break;
				if(len != rclen) continue;
				if(l == rc_l && r == rc_r && hsize(F[i]) + hsize(R[j]) > (uint64_t)p.ihits) {
					F[i].top = F[i].bot = 0; F[i].bwoff = kBwNone; F[i].len = 0;
					R[j].top = R[j].bot = 0; R[j].bwoff = kBwNone; R[j].len = 0;
					break;
				}
			}
		}
	}
	trim_lists(F, nF, R, nR);
}

// Whether a strand list is a raw greedy chain: every hit non-empty and placed, each one ending at or before the next starts.
CFB_HD bool is_chain(const HitRec* L, uint32_t n, uint32_t rdlen) {
	for(uint32_t i = 0; i < n; i++) {
		if(L[i].bwoff == kBwNone || L[i].len == 0 || (uint64_t)L[i].bwoff + L[i].len > rdlen) return false;
		if(i + 1 < n && (uint64_t)L[i].bwoff + L[i].len > L[i + 1].bwoff) return false;
	}
	return true;
}

// post_search for the long hit lists of a long unit, without the nF x nR double loops.  On raw chains (is_chain; otherwise this
// is post_search itself) both loops reduce to the few pairs whose intervals can meet, in the same order:
//  - In read coordinates R[j] covers [rcl_j, rcr_j) with rcl strictly decreasing in j and rcr_j <= rcl_{j-1}.  An extension of
//    R[j] moves only its right end (to the r of the F hit that extended it), and an extension of F[i] only its left end, so rcl
//    stays as it was and every r an earlier F hit had is <= F[i]'s start l.  So at F[i] only R hits whose original interval
//    meets [l, r) pass the two overlap tests: j from the first with rcl_j < r through the first with rcl_j <= l.
//  - The twin loop for F[i] leaves at the first j with rcl_j < l (a zeroed R hit neither leaves nor matches), so only the R hit
//    with rcl_j == l can be its twin.
// rcl: scratch of nR words.
CFB_HDN void post_search_long(const IndexView& v, const Params& p, const uint8_t* fw, uint32_t rdlen,
                              HitRec* F, uint32_t nF, HitRec* R, uint32_t nR, uint32_t* rcl, Counters* ctr) {
	if(!is_chain(F, nF, rdlen) || !is_chain(R, nR, rdlen)) { post_search(v, p, fw, rdlen, F, nF, R, nR, ctr); return; }
	const uint64_t minHitLen = p.min_hitlen;
	uint64_t sum[2] = {0, 0};
	for(uint32_t i = 0; i < nF; i++) if(F[i].len >= minHitLen) sum[0] += F[i].len;
	for(uint32_t i = 0; i < nR; i++) if(R[i].len >= minHitLen) sum[1] += R[i].len;
	if(sum[0] >= minHitLen && sum[1] >= minHitLen) {
		for(uint32_t j = 0; j < nR; j++) rcl[j] = rdlen - R[j].bwoff - R[j].len;
		auto first_below = [&](uint64_t x, bool or_equal) -> uint32_t {     // first j with rcl_j < x (or <= x)
			uint32_t lo = 0, hi = nR;
			while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(rcl[mid] < x || (or_equal && rcl[mid] == x)) hi = mid; else lo = mid + 1; }
			return lo;
		};
		for(uint32_t i = 0; i < nF; i++) {
			const uint64_t len = F[i].len, l = bw64(F[i]), r = l + len;
			const uint32_t j1 = first_below(l, true);
			for(uint32_t j = first_below(r, false); j < nR && j <= j1; j++) {
				const uint64_t rclen = R[j].len;
				if(len < minHitLen && rclen < minHitLen) continue;
				const uint64_t rc_l = (uint64_t)rdlen - bw64(R[j]) - R[j].len, rc_r = rc_l + rclen;
				if(r <= rc_l) continue;
				if(rc_r <= l) continue;
				if(l == rc_l && r == rc_r) continue;
				if(l < rc_l && r > rc_r) continue;
				if(l > rc_l && r < rc_r) continue;
				if(l > rc_l) {
					HitRec t; uint32_t nc; bool dn;
					if(ctr) ctr->ext_searches++;
					partial_search_scalar(v, fw, rdlen, 0, (uint32_t)rc_l, t, nc, dn, ctr);
					if((uint64_t)t.len == len + l - rc_l) F[i] = t;
				}
				if(r > rc_r) {
					HitRec t; uint32_t nc; bool dn;
					if(ctr) ctr->ext_searches++;
					partial_search_scalar(v, fw, rdlen, 1, (uint32_t)((uint64_t)rdlen - r), t, nc, dn, ctr);
					if((uint64_t)t.len == rclen + r - rc_r) R[j] = t;
				}
			}
		}
		for(uint32_t i = 0; i < nF; i++) {
			const uint64_t len = F[i].len, l = bw64(F[i]), r = l + len;
			const uint32_t j = first_below(l, true);
			if(j >= nR || rcl[j] != l || R[j].bwoff == kBwNone) continue;
			const uint64_t rclen = R[j].len, rc_r = l + rclen;
			if(len == rclen && r == rc_r && hsize(F[i]) + hsize(R[j]) > (uint64_t)p.ihits) {
				F[i].top = F[i].bot = 0; F[i].bwoff = kBwNone; F[i].len = 0;
				R[j].top = R[j].bot = 0; R[j].bwoff = kBwNone; R[j].len = 0;
			}
		}
	}
	trim_lists(F, nF, R, nR);
}

// strand choice: returns lo | hi<<1 style pair as (first, second)
CFB_HD void choose_strand(const Params& p, const HitRec* F, uint32_t nF, const HitRec* R, uint32_t nR, int& first, int& second) {
	uint64_t avg[2] = {0, 0}, mx[2] = {0, 0};
	for(int s = 0; s < 2; s++) {
		const HitRec* L = s == 0 ? F : R; const uint32_t n = s == 0 ? nF : nR;
		for(uint32_t i = 0; i < n; i++) {
			const uint64_t len = L[i].len;
			if(len < p.min_hitlen) continue;
			avg[s] += (len - 15) * (len - 15);
			if(len > mx[s]) mx[s] = len;
		}
	}
	if(avg[0] != avg[1]) { first = avg[0] > avg[1] ? 0 : 1; second = first + 1; return; }
	if(mx[0] != mx[1])   { first = mx[0] > mx[1] ? 0 : 1;   second = first + 1; return; }
	first = 0; second = 2;
}

struct HitLess {   // compareBWTHits classifier.h:1058-1086
	CFB_HD bool operator()(const HitRec& a, const HitRec& b) const {
		const uint64_t al = a.len, bl = b.len, as = hsize(a), bs = hsize(b);
		if(al >= 22 || bl >= 22) {
			if(al >= 22 && bl >= 22) { if(as < bs) return true; if(as > bs) return false; }
			if(bl < al) return true;
			if(bl > al) return false;
		}
		if(bl * as < al * bs) return true;
		if(bl * as > al * bs) return false;
		if(as < bs) return true;
		if(as > bs) return false;
		if(bl < al) return true;
		if(bl > al) return false;
		return false;
	}
};

// ----------------------------------------------------------------------------------------
// std::sort as implemented by libstdc++ (bits/stl_algo.h, bits/stl_heap.h): introsort with
// median-of-3 pivot, threshold 16, depth limit 2*floor(log2 n), heapsort fallback, final
// insertion sort.  Restated because the reference's result depends on the exact permutation
// this algorithm produces when the comparator reports ties.
// ----------------------------------------------------------------------------------------
template <class T, class C> CFB_HD void ss_swap(T& a, T& b, C&) { T t = a; a = b; b = t; }

template <class T, class C> CFB_HDN void ss_unguarded_linear_insert(T* last, C comp) {
	T val = *last; T* next = last - 1;
	while(comp(val, *next)) { *last = *next; last = next; --next; }
	*last = val;
}
template <class T, class C> CFB_HDN void ss_insertion_sort(T* first, T* last, C comp) {
	if(first == last) return;
	for(T* i = first + 1; i != last; ++i) {
		if(comp(*i, *first)) { T val = *i; for(T* q = i; q != first; --q) *q = *(q - 1); *first = val; }
		else ss_unguarded_linear_insert(i, comp);
	}
}
template <class T, class C> CFB_HDN void ss_push_heap(T* first, long hole, long top, T value, C comp) {
	long parent = (hole - 1) / 2;
	while(hole > top && comp(first[parent], value)) { first[hole] = first[parent]; hole = parent; parent = (hole - 1) / 2; }
	first[hole] = value;
}
template <class T, class C> CFB_HDN void ss_adjust_heap(T* first, long hole, long len, T value, C comp) {
	const long top = hole; long child = hole;
	while(child < (len - 1) / 2) {
		child = 2 * (child + 1);
		if(comp(first[child], first[child - 1])) child--;
		first[hole] = first[child]; hole = child;
	}
	if((len & 1) == 0 && child == (len - 2) / 2) { child = 2 * (child + 1); first[hole] = first[child - 1]; hole = child - 1; }
	ss_push_heap(first, hole, top, value, comp);
}
template <class T, class C> CFB_HDN void ss_heapsort(T* first, T* last, C comp) {   // __partial_sort(first,last,last)
	long len = (long)(last - first);
	if(len >= 2) {
		long parent = (len - 2) / 2;
		for(;;) { T v = first[parent]; ss_adjust_heap(first, parent, len, v, comp); if(parent == 0) break; parent--; }
	}
	while(last - first > 1) { --last; T v = *last; *last = *first; ss_adjust_heap(first, 0L, (long)(last - first), v, comp); }
}
template <class T, class C> CFB_HDN T* ss_partition_pivot(T* first, T* last, C comp) {
	T* mid = first + (last - first) / 2;
	T *a = first + 1, *b = mid, *c = last - 1;
	if(comp(*a, *b)) { if(comp(*b, *c)) ss_swap(*first, *b, comp); else if(comp(*a, *c)) ss_swap(*first, *c, comp); else ss_swap(*first, *a, comp); }
	else if(comp(*a, *c)) ss_swap(*first, *a, comp);
	else if(comp(*b, *c)) ss_swap(*first, *c, comp);
	else ss_swap(*first, *b, comp);
	T* lo = first + 1; T* hi = last; T* pivot = first;
	for(;;) {
		while(comp(*lo, *pivot)) ++lo;
		--hi;
		while(comp(*pivot, *hi)) --hi;
		if(!(lo < hi)) return lo;
		ss_swap(*lo, *hi, comp);
		++lo;
	}
}
template <class T, class C> CFB_HDN void std_sort(T* first, T* last, C comp) {
	const long n = (long)(last - first);
	if(n <= 0) return;
	if(n > 16) {
		int lg = 0; for(long t = n; t > 1; t >>= 1) lg++;
		// explicit stack instead of recursion: sub-ranges are disjoint, so order is irrelevant
		T* st_first[64]; T* st_last[64]; int st_depth[64]; int sp = 0;
		st_first[0] = first; st_last[0] = last; st_depth[0] = 2 * lg; sp = 1;
		while(sp > 0) {
			--sp; T* f = st_first[sp]; T* l = st_last[sp]; int depth = st_depth[sp];
			while(l - f > 16) {
				if(depth == 0) { ss_heapsort(f, l, comp); break; }
				--depth;
				T* cut = ss_partition_pivot(f, l, comp);
				st_first[sp] = cut; st_last[sp] = l; st_depth[sp] = depth; sp++;
				l = cut;
			}
		}
		ss_insertion_sort(first, first + 16, comp);
		for(T* i = first + 16; i != last; ++i) ss_unguarded_linear_insert(i, comp);
	} else ss_insertion_sort(first, last, comp);
}

// ----------------------------------------------------------------------------------------
// What the rank16 search path leaves out of its hit lists, and when k_prep must put it back.
// nhits[] word of a strand list: hits stored (15 bits) | hits found (15 bits, saturating) << 15 | kListNoLong.  With
// min_hitlen >= kLongLen k_search_t stores only hits of at least kLongLen bases: shorter ones are never counted
// (classifier.h:299), sort after every stored hit (compareBWTHits puts len >= 22 first) and touch nothing else -- unless
// both strands of a mate are in play (extension / twin removal, classifier.h:790-870) or a list is long enough for
// introsort (> 16 hits, where libstdc++'s tie permutation may depend on every element).  In those cases k_prep regenerates
// the full list (list_needs_regen) into a side buffer and points the list at it: word = kListRegen | slot.  Nine of ten hits
// of a typical read are short, so this removes most of the hit traffic and shrinks the per-read device footprint.
// Hits the death bitmap of the K-mer table ends (at most K + 2 bases, only while min_hitlen >= K + 3) are stored with
// top = bot = kUnk, so their size reads as 0; list_needs_exact_ranges says where k_prep must recompute them.
// ----------------------------------------------------------------------------------------
static const uint32_t kListNoLong = 0x80000000u;             // the strand has no hit of min_hitlen bases
static const uint32_t kListRegen = 0x40000000u;              // the list lives in the regeneration buffer, slot = low 30 bits (written by k_prep)
static const uint32_t kLongLen = 22;
CFB_HD uint32_t nh_pack(uint32_t stored, uint32_t found, bool nolong) {
	return (stored & 0x7fffu) | ((found < 0x7fffu ? found : 0x7fffu) << 15) | (nolong ? kListNoLong : 0u);
}
CFB_HD uint32_t nh_stored(uint32_t w) { return w & 0x7fffu; }
CFB_HD uint32_t nh_found(uint32_t w) { return (w >> 15) & 0x7fffu; }

// Whether load_unit empties strand list st of a mate whose nhits words are raw[0], raw[1].  A strand list without a hit of
// min_hitlen bases matters only to the extension step, which needs such a hit on BOTH strands (classifier.h:790-802);
// everything later (trimming within a list, strand choice, counting, scoring) ignores or only shortens short hits.  So unless
// both strands have one, such a list is never read.
CFB_HD bool list_dropped(const uint32_t raw[2], int st) {
	return !((raw[0] | raw[1]) & kListRegen) && (raw[st] & kListNoLong);
}
// Whether k_prep regenerates a list that holds only the long hits: n hits stored, n_other in the mate's other strand list
// (after load_unit), `found` hits found by the search.
CFB_HD bool list_needs_regen(uint32_t n, uint32_t n_other, uint32_t found) {
	return n > 0 && (n_other > 0 || found > 16);
}
// Whether k_prep gives the kUnk hits of a list their exact SA ranges.  A short hit's range can matter
//  - through the twin removal (both strands in play, classifier.h:850-870);
//  - through libstdc++'s tie permutation in lists long enough for introsort (> 16 hits);
//  - through the time stamps, when the list holds a counted hit shorter than kLongLen (only with min_hitlen < 21): such a hit
//    is ordered by size / len among the uncounted short hits (compareBWTHits), so a kUnk hit (size 0) can sort ahead of it.
//    EmitRows advances ts for every hit of a list, counted or not, and after a list left through its `break` the next
//    list's first counted hit shares the previous one's time stamp only at index 0 (kRowSameTs) -- which moves the scores.
// With min_hitlen >= kLongLen - 1 no counted hit is shorter than kLongLen, and the rule is the first two cases alone.
CFB_HD bool list_needs_exact_ranges(const Params& p, const HitRec* L, uint32_t n, uint32_t n_other) {
	if(n == 0) return false;
	if(n_other > 0 || n > 16) return true;
	if(p.min_hitlen + 1 >= kLongLen) return false;
	for(uint32_t i = 0; i < n; i++) if(L[i].len > p.min_hitlen && L[i].len < kLongLen) return true;
	return false;
}

// ----------------------------------------------------------------------------------------
// Resolve planning + scoring
// ----------------------------------------------------------------------------------------
struct UnitHits {      // hit lists of one unit: [mate][strand]
	HitRec* L[2][2]; uint32_t n[2][2]; uint32_t rdlen[2]; int n_mates;
};

// Visit order and per-visit maxGenomeHitSize of go() (classifier.h:228,243-265); calls
// f(rdi, fwi, maxG) for each visited strand list, in order.  Lists must already be post_search'ed.
template <class F> CFB_HDN void for_each_visit(const Params& p, const UnitHits& u, F& f) {
	uint64_t maxG = p.khits;
	for(int rdi = 0; rdi < u.n_mates; rdi++) {
		int a, b;
		choose_strand(p, u.L[rdi][0], u.n[rdi][0], u.L[rdi][1], u.n[rdi][1], a, b);
		for(int fwi = a; fwi < b; fwi++) {
			const HitRec* L = u.L[rdi][fwi]; const uint32_t n = u.n[rdi][fwi];
			for(uint32_t hi = 0; hi < n; hi++) if(L[hi].len >= p.min_hitlen && hsize(L[hi]) > maxG) maxG = hsize(L[hi]);
			if(maxG > p.khits) maxG += p.khits;
			f(rdi, fwi, maxG);
		}
	}
}

struct SortAndCount {   // prep pass: sort each visited list, count rows to resolve
	const Params& p; UnitHits& u; uint64_t rows;
	CFB_HD SortAndCount(const Params& p_, UnitHits& u_) : p(p_), u(u_), rows(0) {}
	CFB_HD void operator()(int rdi, int fwi, uint64_t maxG) {
		HitRec* L = u.L[rdi][fwi]; const uint32_t n = u.n[rdi][fwi];
		std_sort(L, L + n, HitLess());
		uint64_t cnt = 0;
		for(uint32_t hi = 0; hi < n; hi++) {
			if(L[hi].len <= p.min_hitlen) continue;
			if(hsize(L[hi]) == 0) continue;
			const uint64_t nelt = hsize(L[hi]) < maxG ? hsize(L[hi]) : maxG;
			if(nelt > p.ihits) continue;           // resolved-then-discarded in the reference (classifier.h:299)
			rows += nelt; cnt += nelt;
			if(cnt >= maxG) break;
		}
	}
};

struct CountRows {      // same count as SortAndCount on lists that are already sorted (re-run after a capacity overflow)
	const Params& p; const UnitHits& u; uint64_t rows;
	CFB_HD CountRows(const Params& p_, const UnitHits& u_) : p(p_), u(u_), rows(0) {}
	CFB_HD void operator()(int rdi, int fwi, uint64_t maxG) {
		const HitRec* L = u.L[rdi][fwi]; const uint32_t n = u.n[rdi][fwi];
		uint64_t cnt = 0;
		for(uint32_t hi = 0; hi < n; hi++) {
			if(L[hi].len <= p.min_hitlen) continue;
			if(hsize(L[hi]) == 0) continue;
			const uint64_t nelt = hsize(L[hi]) < maxG ? hsize(L[hi]) : maxG;
			if(nelt > p.ihits) continue;
			rows += nelt; cnt += nelt;
			if(cnt >= maxG) break;
		}
	}
};

struct EmitRows {       // second pass: write the SA rows to resolve, in consumption order, with the scoring plan
	const Params& p; const UnitHits& u; uint64_t* out; uint64_t k; uint32_t ts, last_ts;
	uint32_t* hl;           // long units: the whole hit length of every first row (the head keeps 16 bits of it), else null
	CFB_HD EmitRows(const Params& p_, const UnitHits& u_, uint64_t* o, uint32_t* hl_ = nullptr) : p(p_), u(u_), out(o), k(0), ts(0), last_ts(0xffffffffu), hl(hl_) {}
	CFB_HD void operator()(int rdi, int fwi, uint64_t maxG) {
		const HitRec* L = u.L[rdi][fwi]; const uint32_t n = u.n[rdi][fwi];
		uint64_t cnt = 0;
		for(uint32_t hi = 0; hi < n; hi++, ts++) {            // ts advances exactly as in the reference's loop header
			if(L[hi].len <= p.min_hitlen) continue;
			if(hsize(L[hi]) == 0) continue;
			const uint64_t nelt = hsize(L[hi]) < maxG ? hsize(L[hi]) : maxG;
			if(nelt > p.ihits) continue;
			const uint64_t head = kRowStart | ((uint64_t)(L[hi].len & 0xffffu) << 40) | ((uint64_t)(rdi & 1) << 56) | ((uint64_t)(fwi & 1) << 57)
			                    | (ts == last_ts ? kRowSameTs : 0ull);
			last_ts = ts;
			if(hl) hl[k] = L[hi].len;
			for(uint64_t e = 0; e < nelt; e++) out[k++] = ((L[hi].top + e) & kRowMask) | (e == 0 ? head : 0ull);
			cnt += nelt;
			if(cnt >= maxG) break;
		}
	}
};

// Sequence ids are 32-bit, so uniqueID is too; the reference's OFF (a node merged by the tree reduction) is kUidOff, which is
// never below n_seqs.  64 bytes instead of 72 lets k_score keep more hit maps in shared memory.
static const uint32_t kUidOff = 0xffffffffu;
struct Entry {          // HitCount classifier.h:31-57 (fields that influence output)
	uint64_t taxID;
	union {
		uint32_t scores[2][2];
		uint64_t parent;     // once reduce_and_emit has summed the scores: the entry's parent in the current rank round of the tree reduction
	};
	uint32_t lens[2][2];
	uint32_t uniqueID;
	uint32_t score, hitlen, ts;
	int32_t  pid;        // path id or -1 (empty path)
	uint8_t  rank;
	uint8_t  pad[3];
};
struct TaxCnt { uint32_t count; uint32_t pad; uint64_t parent; };
struct TaxCntLess { CFB_HD bool operator()(const TaxCnt& a, const TaxCnt& b) const { return a.count < b.count || (a.count == b.count && a.parent < b.parent); } };

struct OutRec { uint64_t taxid; uint32_t score, hitlen, uid, pad; };   // == cfb_rec

CFB_HD bool is_host(const IndexView& v, uint64_t taxid) {
	uint32_t lo = 0, hi = v.n_host;
	while(lo < hi) { uint32_t mid = (lo + hi) >> 1; if(v.host_taxids[mid] < taxid) lo = mid + 1; else hi = mid; }
	return lo < v.n_host && v.host_taxids[lo] == taxid;
}
CFB_HD uint32_t path_size(const Entry& e) { return e.pid < 0 ? 0u : 10u; }
CFB_HD uint64_t path_at(const IndexView& v, const Entry& e, uint32_t i) {
#ifdef __CUDA_ARCH__
	return __ldg(v.paths + (uint64_t)e.pid * 10 + i);      // read-only for the kernel's life: the loads of a loop may overlap its stores
#else
	return v.paths[(uint64_t)e.pid * 10 + i];
#endif
}

// The record of sequence id `ref` under the context's parameters (score_plan's view of a resolved id): its taxID, or with
// --classification-rank the first non-zero taxID of its path from class_rank_slot on, its path id, whether the exclude set
// holds it, and the rank the resolution stopped at.  With rank > 0 and an empty path the reference's loop
// `for(; rank < path.size(); ...)` does not run and rank keeps its configured value.  cfb_ctx_create tabulates it (IndexView::seqs).
CFB_HD SeqInfo seq_info_of(const IndexView& v, const Params& p, uint32_t ref) {
	SeqInfo s; s.taxid = 0; s.pid = -1;
	uint32_t rank = p.class_rank_slot & 0xffu, excl = 0;
	if(ref < v.n_seqs) {
		s.taxid = v.seq_taxid[ref]; s.pid = v.seq_path[ref];
		excl = v.seq_excluded && v.seq_excluded[ref] ? kSeqExcluded : 0u;
		if(rank > 0 && s.pid >= 0) {
			for(; rank < 10; rank++) { const uint64_t t = v.paths[(uint64_t)s.pid * 10 + rank]; if(t != 0) { s.taxid = t; break; } }
		}
	}
	s.flags = excl | rank << 8;
	return s;
}
CFB_HD SeqInfo seq_info(const IndexView& v, const Params& p, uint32_t ref) {
	if(v.seqs && ref < v.n_seqs) return v.seqs[ref];        // one 16-byte load
	return seq_info_of(v, p, ref);
}

// Third pass: consume the resolved ids along the plan carried by the row words, build the hit map
// (classifier.h:299-345 + addHitToHitMap :982-1050).  Time stamps are non-decreasing along the plan, so "same as the
// previous hit" (kRowSameTs) reproduces every equality the reference's counter produces.  WIDE (long units): the hit length of
// the first row k is hl32[k] (EmitRows' hl), as hits of long reads can exceed the head's 16 bits.
template <bool WIDE = false>
CFB_HDN uint32_t score_plan(const IndexView& v, const Params& p, const uint64_t* rows, const uint32_t* ids, uint64_t n, Entry* map,
                            const uint32_t* hl32 = nullptr) {
	uint32_t nmap = 0, ts = 0;
	for(uint64_t k = 0; k < n;) {
		const uint64_t head = rows[k];
		if(!(head & kRowSameTs)) ts++;
		const uint64_t hl = WIDE ? (uint64_t)hl32[k] : (head >> 40) & 0xffffu; const int rdi = (int)((head >> 56) & 1), fwi = (int)((head >> 57) & 1);
		uint64_t nelt = 1;
		while(k + nelt < n && !(rows[k + nelt] & kRowStart)) nelt++;
		const uint32_t* my = ids + k; k += nelt;
		const uint32_t sc = (uint32_t)((hl - 15) * (hl - 15));
		for(uint64_t e = 0; e < nelt; e++) {
			const uint32_t ref = my[e];
			bool dup = false;                       // coord_ids de-duplication, first-seen order
			for(uint64_t q = 0; q < e; q++) if(my[q] == ref) { dup = true; break; }
			if(dup) continue;
			const SeqInfo si = seq_info(v, p, ref);
			if(si.flags & kSeqExcluded) continue;
			const uint64_t taxID = si.taxid; const int32_t pid = si.pid; const uint8_t rank = (uint8_t)(si.flags >> 8);
			uint32_t idx = 0;
			for(; idx < nmap; ++idx) {
				const bool same = rank == 0 ? (ref == map[idx].uniqueID) : (taxID == map[idx].taxID);
				if(same) {
					if(map[idx].ts != ts) { map[idx].scores[rdi][fwi] += sc; map[idx].lens[rdi][fwi] += (uint32_t)hl; map[idx].ts = ts; }
					break;
				}
			}
			if(idx >= nmap) {
				Entry& n2 = map[nmap++];
				n2.uniqueID = ref; n2.taxID = taxID;
				n2.scores[0][0] = n2.scores[0][1] = n2.scores[1][0] = n2.scores[1][1] = 0;
				n2.lens[0][0] = n2.lens[0][1] = n2.lens[1][0] = n2.lens[1][1] = 0;
				n2.scores[rdi][fwi] = sc; n2.lens[rdi][fwi] = (uint32_t)hl;
				n2.score = 0; n2.hitlen = 0; n2.ts = ts; n2.pid = pid; n2.rank = rank;
			}
		}
	}
	return nmap;
}

// finalize + host rule + tree reduction + emit (classifier.h:380-571).
// map/nmap: hit map; tc: scratch of >= nmap TaxCnt; out: >= nmap records.  Returns #records; *rounds (when given) receives
// the number of rank rounds the tree reduction ran (0: it did not run).
CFB_HDN uint32_t reduce_and_emit(const IndexView& v, const Params& p, bool paired, Entry* map, uint32_t nmap,
                                 TaxCnt* tc, OutRec* out, uint32_t* rounds = nullptr) {
	if(rounds) *rounds = 0;
	const uint32_t k = p.khits;
	for(uint32_t i = 0; i < nmap; i++) {
		Entry& h = map[i];
		const uint32_t s0 = h.scores[0][0] > h.scores[0][1] ? h.scores[0][0] : h.scores[0][1];
		const uint32_t l0 = h.lens[0][0] > h.lens[0][1] ? h.lens[0][0] : h.lens[0][1];
		if(paired) {
			const uint32_t s1 = h.scores[1][0] > h.scores[1][1] ? h.scores[1][0] : h.scores[1][1];
			const uint32_t l1 = h.lens[1][0] > h.lens[1][1] ? h.lens[1][0] : h.lens[1][1];
			h.score = s0 + s1; h.hitlen = l0 + l1;
		} else { h.score = s0; h.hitlen = l0; }
	}
	int64_t best = 0; bool only_host = false;
	for(uint32_t i = 0; i < nmap; i++) {
		if((int64_t)map[i].score > best) { best = map[i].score; only_host = is_host(v, map[i].taxID); }
		else if((int64_t)map[i].score == best) only_host |= is_host(v, map[i].taxID);
	}
	if(!only_host && nmap > k) {
		uint32_t bs = map[0].score;
		for(uint32_t i = 1; i < nmap; i++) if(bs < map[i].score) bs = map[i].score;
		for(int i = 0; i < (int)nmap; i++) {
			if(map[i].score < bs) { if(i + 1 < (int)nmap) map[i] = map[nmap - 1]; nmap--; i--; }
		}
		if(!p.tree_traverse && nmap > k) return 0;
		uint8_t rank = 0;
		while(nmap > k) {
			if(rounds) *rounds += 1;
			// every entry of this round gets its parent once, with loads that do not wait for each other; the tc loop below
			// compares against the stored value
			for(uint32_t i = 0; i < nmap; i++) {
				Entry& h = map[i];
				while(h.rank < rank) {
					if((uint32_t)h.rank + 1 >= path_size(h)) { h.rank = 255; break; }
					h.rank += 1; h.taxID = path_at(v, h, h.rank);
				}
				if(h.rank == rank) h.parent = ((uint32_t)rank + 1 >= path_size(h)) ? 1 : path_at(v, h, rank + 1);
			}
			uint32_t ntc = 0;
			for(uint32_t i = 0; i < nmap; i++) {
				const Entry& h = map[i];
				if(h.rank != rank) continue;
				const uint64_t parent = h.parent;
				if(parent == 0) continue;
				uint32_t j = 0;
				for(; j < ntc; j++) if(tc[j].parent == parent) { tc[j].count += 1; break; }
				if(j == ntc) { tc[ntc].count = 1; tc[ntc].pad = 0; tc[ntc].parent = parent; ntc++; }
			}
			if(ntc == 0) {
				if(rank < path_size(map[0])) { rank++; continue; } else break;
			}
			ss_heapsort(tc, tc + ntc, TaxCntLess());    // keys are distinct: any correct sort gives std::sort's result
			uint32_t j = ntc;
			while(j-- > 0) {
				const uint64_t parent = tc[j].parent;
				for(uint32_t i = 0; i < nmap; i++) {
					Entry& h = map[i];
					if(h.rank == rank && h.parent == parent) { h.uniqueID = kUidOff; h.rank = rank + 1; h.taxID = parent; }
				}
				bool first = true;
				for(uint32_t i = 0; i < nmap; i++) {
					if(parent == map[i].taxID) {
						if(!first) { if(i + 1 < nmap) map[i] = map[nmap - 1]; nmap--; i--; }
						else first = false;
					}
				}
				if(nmap <= k) break;
			}
			++rank;
			if(rank > path_size(map[0])) break;
		}
	}
	if(!only_host && nmap > k) return 0;
	uint32_t no = 0;
	for(uint32_t i = 0; i < nmap; i++) {
		if(only_host && !is_host(v, map[i].taxID)) continue;
		OutRec r; r.taxid = map[i].taxID; r.score = map[i].score; r.hitlen = map[i].hitlen;
		r.uid = map[i].uniqueID < v.n_seqs ? map[i].uniqueID : 0xFFFFFFFFu; r.pad = 0;
		out[no++] = r;
	}
	return no;
}

// Scalar resolve of one SA row (walk-left to a sampled / boundary / '$' row; no "+steps",
// group_walk.h:508-512; tryOffset bt2_idx.h:1980-2014).  Scalar twin of k_resolve_c.
CFB_HDN uint32_t resolve_scalar(const IndexView& v, uint64_t row, Counters* ctr) {
	const uint64_t lowmask = ((uint64_t)1 << v.off_rate) - 1;
	for(;;) {
		if(row == v.zoff) return 0;
		if((row & lowmask) == 0) {
			const uint64_t i = row >> v.off_rate;
			return v.sample32 ? v.sample32[i] : (uint32_t)v.sample16[i];
		}
		if(v.n_boundaries && row <= v.last_boundary) {
			const uint64_t b = row >> v.bshift;
			if(v.bbits[b >> 5] & (1u << (b & 31))) {
				uint32_t lo = 0, hi = v.n_boundaries;
				while(lo < hi) { uint32_t mid = (lo + hi) >> 1; if(v.brow[mid] < row) lo = mid + 1; else hi = mid; }
				if(lo < v.n_boundaries && v.brow[lo] == row) return v.sample32 ? v.bseq[lo] : (uint32_t)(uint16_t)v.bseq[lo];
			}
		}
		row = lf_scalar(v, row, bwt_char(v, row));
		if(ctr) ctr->walk_steps++;
	}
}

}  // namespace cfb
#endif
