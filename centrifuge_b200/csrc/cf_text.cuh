// cf_text.cuh -- text-level operator (SURVEY.md 8f rank 1): FASTQ/FASTA bytes -> classification TSV,
// everything between the file read and the file write on the device.  Included at the end of
// cfb200.cu (it uses Slot / enqueue_kernels / finish_batch and the scan kernels).
//
// Reference semantics restated (paths relative to the reference tree):
//   record layout, base/quality handling      pat.cpp:725-849 (FASTA), :852-1157 (FASTQ)
//   per-read seed                              pat.h:55-91 (genRandSeed)
//   N / length filters                         centrifuge.cpp:2550-2596, aligner_seed_policy.cpp:296-298
//   AlnSetSumm best / second best              aligner_result.h:398-427
//   selectByScore + shufflePortion             aln_sink.h:1861-1927, ds.h:784-795, random_source.h:34-61
//   row text                                   aln_sink.h:2202-2337
//   SpeciesMetrics::addSpeciesCounts           aln_sink.h:142-172
// Only the *strict* layout is handled here (one line per field, LF line ends); every deviation raises a
// status bit and the caller re-does the span with the byte-exact host state machine in cf_host.cpp.
//
// Stages per span (all on the slot's stream):
//   k_nl_count / scan / k_nl_write   positions of all line ends (16-byte loads, SIMD byte compare)
//   k_tok_rec                        thread per (record, mate): line spans, lengths after trimming
//   [k_tok_quals]                    warp per unit, only for FASTQ in another encoding than phred33: qualities checked
//                                    and converted to phred33 into a side buffer (the uploaded text stays as it is)
//   scan                             base offsets
//   k_tok_bases                      warp per unit: ASCII -> codes (coalesced), N filter, seed hash
//   [classification kernels of cfb200.cu, unchanged]
//   k_fmt_plan                       thread per unit: best/second, tie selection with the per-read LCG,
//                                    row byte counts, per-taxon counters (warp-aggregated atomics)
//   scan                             text offsets
//   k_fmt_write                      CTA per 128 units: rows composed in shared memory, coalesced store; CTAs whose
//                                    rows do not fit (sequence / quality columns) write warp per unit, the warp
//                                    copying long fields together
// Rows follow the context's column list (cfb_ctx_set_columns, --tab-fmt-cols) through the row composer of cf_cols.h,
// the same one the host formatter uses.

#include "cf_cols.h"
#include "cf_nceil.h"
#include "cf_quals.h"

enum { TX_IRREGULAR = 1, TX_LINECOUNT = 2, TX_FMT_OVERFLOW = 4 };
static const int kFmtMax = 32;          // records per unit the on-device selector holds
static const int kTextTile = 4096;      // bytes per CTA of the line-end kernels (256 threads x 16 B)

struct TextArgs {
	const uint8_t* text[2]; uint32_t nbytes[2];
	uint32_t* nl[2]; const uint64_t* nl_total[2];
	uint32_t n_rec; int32_t lines_per, n_mates, fasta, trim5, trim3; uint32_t seed;
	uint32_t* len[2]; uint64_t* off[2]; uint8_t* flags; uint32_t* seedv[2]; uint32_t maxlen_hint;
	uint32_t keep_long;             // 0: a unit with a mate over kLongUnitLen bases gets flags 0 (the span is run again with the long-unit kernels)
	uint32_t* name_off; uint32_t* id_len; uint32_t* name_len; uint32_t* seq_off[2]; uint32_t* qual_off[2];
	uint8_t* bases;
	unsigned long long* tscal;      // [0] status bits, [1] max length, [2] n_multi, [3] max length of the mates up to kLongUnitLen bases
	int32_t nc_type; double nc_c, nc_l, nc_mn, nc_mx;      // N ceiling (cf_nceil.h)
	int32_t q_bits; uint32_t sol_steps;                     // quality encoding (cf_quals.h QualBits; 0: phred33) and Solexa steps
	uint8_t* qconv[2];              // k_tok_quals' phred33 qualities, at the offsets of the quality line (q_bits != 0)
	const uint8_t* qtext[2];        // where k_tok_bases<true> reads the qualities (qconv)
};

// 16-bit mask of bytes equal to `c` in a 16-byte vector
__device__ __forceinline__ uint32_t eq_mask16(const uint4 v, uint32_t c4) {
	uint32_t r = 0;
	const uint32_t w[4] = {v.x, v.y, v.z, v.w};
	#pragma unroll
	for(int k = 0; k < 4; k++) {
		const uint32_t m = __vcmpeq4(w[k], c4) & 0x01010101u;
		r |= ((m & 1u) | ((m >> 7) & 2u) | ((m >> 14) & 4u) | ((m >> 21) & 8u)) << (4 * k);
	}
	return r;
}
__device__ __forceinline__ uint32_t tile_masks(const uint8_t* text, uint32_t nbytes, uint32_t& cr) {
	const uint32_t pos = blockIdx.x * kTextTile + threadIdx.x * 16;
	uint32_t m = 0; cr = 0;
	if(pos < nbytes) {
		const uint4 v = *reinterpret_cast<const uint4*>(text + pos);
		const uint32_t valid = nbytes - pos >= 16 ? 0xffffu : ((1u << (nbytes - pos)) - 1u);
		m = eq_mask16(v, 0x0a0a0a0au) & valid;
		cr = eq_mask16(v, 0x0d0d0d0du) & valid;
	}
	return m;
}
__global__ void __launch_bounds__(256) k_nl_count(const uint8_t* text, uint32_t nbytes, uint32_t* tile_cnt, unsigned long long* tscal) {
	__shared__ uint32_t sh[8];
	uint32_t cr; const uint32_t m = tile_masks(text, nbytes, cr);
	uint32_t c = __popc(m);
	if(__any_sync(0xffffffffu, cr != 0) && (threadIdx.x & 31) == 0) atomicOr(tscal, (unsigned long long)TX_IRREGULAR);   // CR anywhere: not the strict layout
	for(int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
	if((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
	__syncthreads();
	if(threadIdx.x == 0) { uint32_t s = 0; for(int i = 0; i < 8; i++) s += sh[i]; tile_cnt[blockIdx.x] = s; }
}
__global__ void __launch_bounds__(256) k_nl_write(const uint8_t* text, uint32_t nbytes, const uint64_t* tile_off, uint32_t* nl, uint64_t cap) {
	__shared__ uint32_t sh[8];
	uint32_t cr; uint32_t m = tile_masks(text, nbytes, cr);
	const uint32_t c = __popc(m);
	uint32_t incl = c;
	const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	for(int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if((int)lane >= d) incl += t; }
	if(lane == 31) sh[w] = incl;
	__syncthreads();
	uint32_t wbase = 0;
	for(uint32_t i = 0; i < w; i++) wbase += sh[i];
	uint64_t o = tile_off[blockIdx.x] + wbase + incl - c;
	const uint32_t pos = blockIdx.x * kTextTile + threadIdx.x * 16;
	while(m) { const int b = __ffs(m) - 1; m &= m - 1; if(o < cap) nl[o] = pos + b; o++; }
}

__device__ __forceinline__ uint32_t trimmed_len(uint32_t nread, int trim5, int trim3) {
	uint32_t l = nread > (uint32_t)trim5 ? nread - trim5 : 0;
	return l > (uint32_t)trim3 ? l - trim3 : 0;
}

// thread per (record, mate): line spans of the strict layout
__global__ void __launch_bounds__(128) k_tok_rec(const TextArgs a) {
	const uint64_t i = (uint64_t)blockIdx.x * 128 + threadIdx.x;
	if(i >= (uint64_t)a.n_rec * a.n_mates) return;
	const int m = (int)(i / a.n_rec); const uint32_t r = (uint32_t)(i % a.n_rec);
	const uint32_t L = a.lines_per;
	a.len[m][r] = 0;
	if(*a.nl_total[m] != (uint64_t)a.n_rec * L) { if(r == 0) atomicOr(a.tscal, (unsigned long long)TX_LINECOUNT); return; }
	const uint32_t* nl = a.nl[m]; const uint8_t* t = a.text[m];
	const uint32_t j0 = r * L;
	const uint32_t s0 = j0 ? nl[j0 - 1] + 1 : 0, e0 = nl[j0], s1 = e0 + 1, e1 = nl[j0 + 1];
	bool bad = e0 <= s0 + 1 || t[s0] != (a.fasta ? '>' : '@');       // marker + non-empty name
	const uint32_t nread = e1 - s1;
	bad |= nread == 0;
	uint32_t qoff = 0;
	if(!a.fasta) {
		const uint32_t s2 = e1 + 1, e2 = nl[j0 + 2], s3 = e2 + 1, e3 = nl[j0 + 3];
		bad |= e2 == s2 || t[s2] != '+';
		// kept qualities (from trim5 on, minus trim3) must cover the read and may be one longer (pat.cpp:1073-1078)
		const uint32_t kept = trimmed_len(e3 - s3, a.trim5, a.trim3), want = trimmed_len(nread, a.trim5, a.trim3);
		if(!(a.q_bits & QUAL_INTEGER)) bad |= kept < want || kept > want + 1;      // integer qualities: k_tok_quals counts them
		qoff = s3;
	}
	if(bad) { atomicOr(a.tscal, (unsigned long long)TX_IRREGULAR); return; }
	const uint32_t len = trimmed_len(nread, a.trim5, a.trim3);
	if((unsigned long long)len > *(volatile unsigned long long*)(a.tscal + 1)) atomicMax(a.tscal + 1, (unsigned long long)len);   // guarded: one address for all records
	if(len <= kLongUnitLen && (unsigned long long)len > *(volatile unsigned long long*)(a.tscal + 3)) atomicMax(a.tscal + 3, (unsigned long long)len);
	// the short kernels' buffers are sized for the hint: the host re-runs the span with a wider class.  Long mates are laid out
	// by their own lengths, like every mate, and classified by the long-unit kernels.
	if(len > a.maxlen_hint && len <= kLongUnitLen) return;
	a.len[m][r] = len;
	a.seq_off[m][r] = s1; a.qual_off[m][r] = qoff;
	if(m == 0) { a.name_off[r] = s0 + 1; a.name_len[r] = e0 - s0 - 1; }
	else a.seedv[1][r] = e0 - s0 - 1;          // mate-2 name length, replaced by the seed in k_tok_bases
}

__device__ __forceinline__ bool is_alpha(uint32_t c) { const uint32_t l = c | 0x20u; return l >= 'a' && l <= 'z'; }
__device__ __forceinline__ bool is_dnacat(uint32_t c) {     // asc2dnacat > 0 (alphabet.cpp:36-58) or '-'
	if(c == '-') return true;
	const uint32_t l = c | 0x20u;
	if(l < 'a' || l > 'z') return false;
	return (0x01ee34cfu >> (l - 'a')) & 1u;                  // a b c d g h k m n r s t v w x y
}
__device__ __forceinline__ uint32_t dna_code(uint32_t c) {
	const uint32_t l = c | 0x20u;
	return l == 'c' ? 1u : (l == 'g' ? 2u : (l == 't' ? 3u : (l == 'n' ? 4u : 0u)));
}
__device__ __forceinline__ uint32_t warp_xor(uint32_t x) { for(int d = 16; d > 0; d >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, d); return x; }
__device__ __forceinline__ uint32_t warp_add(uint32_t x) { for(int d = 16; d > 0; d >>= 1) x += __shfl_xor_sync(0xffffffffu, x, d); return x; }
__device__ __forceinline__ bool is_space(uint32_t c) { return c == ' ' || (c >= 9 && c <= 13); }

// warp per unit: bases, N filter, seeds, read id length.  kConv: the qualities are k_tok_quals' phred33 bytes in
// qtext (another encoding); the phred33 instance reads them from the text and is the kernel it always was.
template <bool kConv>
__global__ void __launch_bounds__(128, 16) k_tok_bases(const TextArgs a) {      // latency-bound: all 64 warp slots of an SM
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t u = blockIdx.x * 4 + (threadIdx.x >> 5);
	if(u >= a.n_rec) return;
	if((*a.tscal & (TX_IRREGULAR | TX_LINECOUNT)) || a.tscal[3] > a.maxlen_hint) return;
	uint32_t flags = 0; bool bad = false;
	const uint64_t total0 = a.off[0][a.n_rec];
	for(int m = 0; m < a.n_mates; m++) {
		const uint8_t* t = a.text[m];
		const uint8_t* qt = kConv ? a.qtext[m] : t;
		const uint32_t len = a.len[m][u], so = a.seq_off[m][u], qo = a.qual_off[m][u];
		const uint32_t line = a.nl[m][u * a.lines_per + 1] - so;
		const uint32_t nlen = m == 0 ? a.name_len[u] : a.seedv[1][u];
		const uint32_t no = so - 1 - nlen;
		const uint64_t boff = a.off[m][u] + (m ? total0 : 0ull);
		__syncwarp();
		if(m == 1 && lane == 0) a.off[1][u] = boff;         // BatchView offsets are absolute
		uint8_t* dst = a.bases + boff;
		uint32_t sx = 0, ns = 0;
		for(uint32_t i4 = lane * 4; i4 < line; i4 += 128) {          // 4 characters per lane
			const uint32_t v = load4(t, (uint64_t)so + i4);
			uint32_t codes = 0, nvalid = 0;
			#pragma unroll
			for(uint32_t b = 0; b < 4; b++) {
				const uint32_t i = i4 + b;
				if(i >= line) break;
				uint32_t c = (v >> (8 * b)) & 0xffu;
				if(a.fasta) { if(!is_dnacat(c)) bad = true; }
				else { if(c == '.') c = 'N'; if(!is_alpha(c)) bad = true; }
				const uint32_t code = dna_code(c);
				if(i >= (uint32_t)a.trim5 && i - a.trim5 < len) {
					const uint32_t j = i - a.trim5;
					codes |= code << (8 * b); nvalid++;
					sx ^= code << ((j & 15) << 1);
					ns += code == 4;
				}
			}
			if(nvalid == 4 && ((boff + (i4 - a.trim5)) & 3ull) == 0) *reinterpret_cast<uint32_t*>(dst + (i4 - a.trim5)) = codes;
			else for(uint32_t b = 0; b < 4; b++) { const uint32_t i = i4 + b; if(i < line && i >= (uint32_t)a.trim5 && i - a.trim5 < len) dst[i - a.trim5] = (uint8_t)(codes >> (8 * b)); }
		}
		if(a.fasta) {                                        // every FASTA base has quality 'I' (pat.cpp:828)
			for(uint32_t j = lane; j < len; j += 32) sx ^= (uint32_t)'I' << ((j & 3) << 3);
		} else {
			for(uint32_t j4 = lane * 4; j4 < len; j4 += 128) {    // quality contribution: byte (j & 3) of the seed word
				const uint32_t v = load4(qt, (uint64_t)qo + a.trim5 + j4);
				const uint32_t keep = len - j4 >= 4 ? 0xffffffffu : ((1u << (8 * (len - j4))) - 1u);
				sx ^= v & keep;
			}
			// phred33 characters only (qual.h:136-142; a space is an error too).  In another encoding k_tok_quals wrote
			// phred33 bytes over the whole line (the converted ones, 'I' elsewhere), so the check only catches what it let
			// through: bytes past 127, which the seed would read as negative chars, go to the host reader.
			const uint32_t qlen = a.nl[m][u * a.lines_per + 3] - qo;
			for(uint32_t j4 = lane * 4; j4 < qlen; j4 += 128) {
				const uint32_t v = load4(qt, (uint64_t)qo + j4);
				const uint32_t keep = qlen - j4 >= 4 ? 0xffffffffu : ((1u << (8 * (qlen - j4))) - 1u);
				if((__vcmpltu4(v, 0x21212121u) | __vcmpgtu4(v, 0x7f7f7f7fu)) & keep) bad = true;
			}
		}
		// name: up to the first '/' (pat.h:84-88); chars are signed in the reference
		bool slashed = false;
		for(uint32_t base = 0; base < nlen && (!slashed || a.fasta); base += 32) {
			const uint32_t i = base + lane;
			const uint32_t c = i < nlen ? t[no + i] : 0;
			if(a.fasta && c == '>') bad = true;              // a '>' inside the name line ends the name in the reference parser
			if(!slashed) {
				const uint32_t slash = __ballot_sync(0xffffffffu, i < nlen && c == '/');
				const uint32_t before = slash ? ((1u << (__ffs(slash) - 1)) - 1u) : 0xffffffffu;
				if(i < nlen && ((before >> lane) & 1u)) sx ^= ((uint32_t)(int32_t)(int8_t)c) << ((i & 3) << 3);
				slashed = slash != 0;
			}
		}
		sx = warp_xor(sx); ns = warp_add(ns);
		const uint32_t rseed = ((a.seed + 101u) * 59u * 61u * 67u * 71u * 73u * 79u * 83u) ^ sx;
		bool pass = len >= 2;
		if(pass) { bool sure; pass = nceil_pass(a.nc_type, a.nc_c, a.nc_l, a.nc_mn, a.nc_mx, len, ns, &sure); if(!sure) bad = true; }   // a log ceiling the device cannot settle: the span goes to the host reader
		if(pass) flags |= 1u << m;
		if(lane == 0) a.seedv[m][u] = (m == 1 && len == 0) ? 0u : rseed;
		if(m == 0) {   // read id: drop a trailing /1 /2 /3, cut at the first whitespace (aln_sink.h:2202-2217)
			uint32_t n2 = nlen;
			if(nlen >= 2 && t[no + nlen - 2] == '/') { const uint32_t d = t[no + nlen - 1]; if(d == '1' || d == '2' || d == '3') n2 = nlen - 2; }
			uint32_t idl = n2;
			for(uint32_t base = 0; base < n2; base += 32) {
				const uint32_t i = base + lane;
				const uint32_t sp = __ballot_sync(0xffffffffu, i < n2 && is_space(t[no + i]));
				if(sp) { idl = base + __ffs(sp) - 1; break; }
			}
			if(lane == 0) a.id_len[u] = idl;
		}
	}
	if(__any_sync(0xffffffffu, bad)) { if(lane == 0) atomicOr(a.tscal, (unsigned long long)TX_IRREGULAR); }
	if(lane == 0) {
		const bool long_unit = !a.keep_long && (a.len[0][u] > kLongUnitLen || (a.n_mates == 2 && a.len[1][u] > kLongUnitLen));
		a.flags[u] = long_unit ? (uint8_t)0 : (uint8_t)flags;
	}
}

// warp per unit, FASTQ in another encoding than phred33 (cf_quals.h): every mate's quality line checked and converted
// to phred33 into qconv at the line's own offsets, so that k_tok_bases and the formatter read it where they would read
// the text.  Whatever the reference refuses, and whatever this kernel does not settle exactly, marks the span irregular
// and the record-level reader decides it (with the reference's message where it is an error).
//   character qualities (pat.cpp:1042-1078): a space anywhere is refused; the characters from trim5 on are converted
//     (solexa, else phred64 refusing c < 64); the ones before trim5 are neither checked nor printed ('I' is stored)
//   integer qualities (pat.cpp:997-1030): token starts by ballots over the line (the first byte always starts one, an
//     empty one when it is a space; after that every non-space after a space), each token parsed by the lane at its
//     start as atoi does; the count of kept tokens must cover the read and may be one longer.  To the host: a line of
//     4095 bytes or more (FileBuf::gets splits it), a NUL, more than 9 digits, a negative value, and a Solexa value
//     whose phred33 byte passes 127.  Past the converted values the line is filled with 'I'.
__global__ void __launch_bounds__(128) k_tok_quals(const TextArgs a) {
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t u = blockIdx.x * 4 + (threadIdx.x >> 5);
	if(u >= a.n_rec) return;
	if((*a.tscal & (TX_IRREGULAR | TX_LINECOUNT)) || a.tscal[3] > a.maxlen_hint) return;
	const bool solexa = a.q_bits & QUAL_SOLEXA, phred64 = a.q_bits & QUAL_PHRED64;
	bool bad = false;
	for(int m = 0; m < a.n_mates; m++) {
		const uint32_t* nl = a.nl[m] + (uint64_t)u * 4;
		const uint32_t s3 = nl[2] + 1, qlen = nl[3] - s3, nread = nl[1] - nl[0] - 1;
		const uint8_t* t = a.text[m] + s3; uint8_t* q = a.qconv[m] + s3;
		if(!(a.q_bits & QUAL_INTEGER)) {
			for(uint32_t i = lane; i < qlen; i += 32) {
				const uint32_t c = t[i];
				int v = 'I';
				if(c == ' ') bad = true;
				else if(i >= (uint32_t)a.trim5) { v = qual_from_char(c, solexa, phred64, a.sol_steps); if(v < 0) bad = true; }
				q[i] = (uint8_t)v;
			}
			continue;
		}
		if(qlen >= 4095) { bad = true; continue; }
		uint32_t count = 0;
		for(uint32_t base = 0; base < qlen; base += 32) {
			const uint32_t i = base + lane;
			const uint32_t c = i < qlen ? t[i] : ' ';
			if(i < qlen && c == 0) bad = true;
			const bool start = i < qlen && (i == 0 || (c != ' ' && t[i - 1] == ' '));
			const uint32_t starts = __ballot_sync(0xffffffffu, start);
			if(start) {
				int v = 0;                                   // the empty first token of a line that starts with a space reads as 0
				if(c != ' ') {
					uint32_t p = i;
					while(p < qlen && t[p] >= 9 && t[p] <= 13) p++;
					bool neg = false;
					if(p < qlen && (t[p] == '+' || t[p] == '-')) { neg = t[p] == '-'; p++; }
					for(uint32_t nd = 0; p < qlen && t[p] >= '0' && t[p] <= '9'; p++) {
						if(++nd > 9) { bad = true; break; }
						v = v * 10 + (int)(t[p] - '0');
					}
					if(neg) v = -v;
				}
				const int pq = qual_from_int(v, solexa, a.sol_steps);
				if(pq < 33 || pq > 127) bad = true;
				q[count + __popc(starts & ((1u << lane) - 1u))] = (uint8_t)pq;
			}
			count += __popc(starts);
		}
		if(trimmed_len(count, a.trim5, a.trim3) < trimmed_len(nread, a.trim5, a.trim3) ||
		   trimmed_len(count, a.trim5, a.trim3) > trimmed_len(nread, a.trim5, a.trim3) + 1) bad = true;
		for(uint32_t i = count + lane; i < qlen; i += 32) q[i] = 'I';
	}
	if(__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(a.tscal, (unsigned long long)TX_IRREGULAR);
}

// ------------------------------------------------------------------------------ formatter
struct FmtTables {
	const uint64_t* nd_taxid; const uint8_t* nd_info; uint32_t n_nodes;       // info = rank | leaf << 7
	const uint64_t* sp_taxid; uint32_t n_sp;
	const uint32_t* sn_off; const char* sn_blob; uint32_t n_seq;              // sequence names
	const uint64_t* nm_taxid; const uint32_t* nm_off; const char* nm_blob; uint32_t n_names;   // taxon names (taxName), ascending taxid
	const uint8_t* rk_off; const char* rk_blob;                               // rank strings, RANK_MAX + 1 offsets
};
struct FmtArgs {
	FmtTables tb;
	const uint8_t* text; const uint32_t* name_off; const uint32_t* id_len;
	const uint32_t* len[2]; const uint8_t* flags; const uint32_t* seedv[2];
	const uint32_t* rec_off; const OutRec* recs; uint32_t n_units; int32_t n_mates; uint32_t khits;
	uint32_t* row_bytes; const uint64_t* txt_off; uint8_t* sel; uint8_t* num; uint32_t* sec;
	char* out; uint64_t out_cap;
	unsigned long long* sp; unsigned long long* multi; uint32_t multi_stride; uint64_t multi_cap;
	unsigned long long* tscal; uint32_t maxlen_hint;
	const uint8_t* cols; uint32_t n_cols, col_mask;                          // column list (device copy) and its field mask
	const uint8_t* qtext[2]; const uint8_t* bases; const uint64_t* off[2];   // sequence / quality columns: trimmed codes, phred33 qualities
	const uint32_t* qual_off[2]; const uint32_t* nl[2]; int32_t lines_per, fasta, trim5, trim3;
	int32_t q_int;                  // integer qualities: the kept values are cut to the read's length
};
// A span the tokeniser rejected (or that needs a wider length class) has no valid name / id / flag arrays: the
// formatter must not touch them.  The bits tested here are final before the formatter starts.
__device__ __forceinline__ bool span_rejected(const FmtArgs& a) {
	return (*(volatile unsigned long long*)a.tscal & (TX_IRREGULAR | TX_LINECOUNT)) != 0 || *(volatile unsigned long long*)(a.tscal + 3) > a.maxlen_hint;
}

__device__ __forceinline__ int find_u64(const uint64_t* a, uint32_t n, uint64_t key) {
	uint32_t lo = 0, hi = n;
	while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(a[mid] < key) lo = mid + 1; else hi = mid; }
	return (lo < n && a[lo] == key) ? (int)lo : -1;
}
// The record's fields of a row: seqID (classifier.h:557 + appendSeqID aln_sink.h:2220-2234), taxRank (the node's rank,
// rank 0 for unclassified rows, classifier.h:540-546,619-626), taxName (name table, "" by default) and the numbers.
__device__ __forceinline__ void rec_row(const FmtArgs& a, bool uncl, const OutRec* r, ColRow& row) {
	const FmtTables& tb = a.tb;
	uint64_t taxid = 0; uint32_t uid = 0xffffffffu;
	row.score = 0; row.hitlen = 0;
	if(!uncl) { taxid = r->taxid; row.score = r->score; row.hitlen = r->hitlen; uid = r->uid; }
	row.taxid = taxid;
	int rank = 0;
	if(uncl) { row.sid = tb.rk_blob + tb.rk_off[RANK_MAX]; row.sl = 12; }
	else {
		const int nd = find_u64(tb.nd_taxid, tb.n_nodes, taxid);
		const bool leaf = nd >= 0 ? (tb.nd_info[nd] >> 7) != 0 : true;
		rank = nd >= 0 ? (tb.nd_info[nd] & 0x7f) : 0;
		if(leaf && uid != 0xffffffffu && uid < tb.n_seq) { row.sid = tb.sn_blob + tb.sn_off[uid]; row.sl = tb.sn_off[uid + 1] - tb.sn_off[uid]; }
		else { row.sid = tb.rk_blob + tb.rk_off[rank]; row.sl = (uint32_t)tb.rk_off[rank + 1] - tb.rk_off[rank]; }
	}
	row.rank = tb.rk_blob + tb.rk_off[rank]; row.rl = (uint32_t)tb.rk_off[rank + 1] - tb.rk_off[rank];
	row.name = tb.rk_blob; row.nl = 0;
	if(a.col_mask & (1u << COL_TAX_NAME)) {
		const int k = find_u64(tb.nm_taxid, tb.n_names, taxid);
		if(k >= 0) { row.name = tb.nm_blob + tb.nm_off[k]; row.nl = tb.nm_off[k + 1] - tb.nm_off[k]; }
	}
}
// The unit's fields of a row: read ID, query length, and the mates' trimmed bases and kept qualities when printed.
__device__ __forceinline__ void unit_row(const FmtArgs& a, uint32_t u, ColRow& row) {
	row.id = (const char*)a.text + a.name_off[u]; row.idl = a.id_len[u];
	row.paired = a.n_mates == 2;
	for(int m = 0; m < 2; m++) { row.seq[m] = a.bases; row.len[m] = 0; row.qual[m] = nullptr; row.qn[m] = 0; }
	for(int m = 0; m < a.n_mates; m++) {
		row.len[m] = a.len[m][u];
		if(a.col_mask & kColSeqBits) row.seq[m] = a.bases + a.off[m][u];        // k_tok_bases wrote the codes there
		if(a.col_mask & kColQualBits) {
			if(a.fasta) row.qn[m] = row.len[m];                                  // all 'I' (pat.cpp:828)
			else {     // the quality line from trim5 on, minus trim3: as long as the read or one longer (pat.cpp:1072-1078);
				       // integer qualities are cut to the read's length (pat.cpp:1024-1027)
				const uint32_t qo = a.qual_off[m][u];
				row.qn[m] = a.q_int ? row.len[m] : trimmed_len(a.nl[m][u * a.lines_per + 3] - qo, a.trim5, a.trim3);
				row.qual[m] = (const char*)a.qtext[m] + qo + a.trim5;
			}
		}
	}
	row.qlen = (uint64_t)row.len[0] + row.len[1];
}
// warp-cooperative byte sink: every lane holds the same cursor, long fields are copied with one byte per lane and step
// (coalesced loads and stores), numbers and single characters are written by lane 0
struct ColWarpWriter {
	char* p; uint32_t lane;
	__device__ __forceinline__ void put(char c) { if(lane == 0) *p = c; p++; }
	__device__ __forceinline__ void copy(const char* s, uint32_t k) { for(uint32_t i = lane; i < k; i += 32) p[i] = s[i]; p += k; }
	__device__ __forceinline__ void fill(char c, uint32_t k) { for(uint32_t i = lane; i < k; i += 32) p[i] = c; p += k; }
	__device__ __forceinline__ void bases(const uint8_t* b, uint32_t k) { for(uint32_t i = lane; i < k; i += 32) p[i] = "ACGTN"[b[i]]; p += k; }
	__device__ __forceinline__ void num(uint64_t v) { if(lane == 0) { ColWriter w; w.p = p; w.num(v); } p += col_digits(v); }
};
struct Lcg32 { uint32_t last; __device__ __forceinline__ uint32_t next() { last = 1664525u * last + 1013904223u; const uint32_t r = last >> 16; last = 1664525u * last + 1013904223u; return r ^ last; } };

__global__ void __launch_bounds__(128) k_fmt_plan(const FmtArgs a) {
	const uint32_t u = blockIdx.x * 128 + threadIdx.x;
	const bool live = u < a.n_units;
	if(span_rejected(a)) { if(live) a.row_bytes[u] = 0; return; }
	uint32_t r0 = 0, r1 = 0;
	if(live) { r0 = a.rec_off[u]; r1 = a.rec_off[u + 1]; }
	const bool uncl = r1 == r0;
	const uint32_t sz = uncl ? 1u : r1 - r0;
	bool ok = live;
	if(live && sz > (uint32_t)kFmtMax) { atomicOr(a.tscal, (unsigned long long)TX_FMT_OVERFLOW); a.row_bytes[u] = 0; ok = false; }
	uint32_t sc[kFmtMax]; uint8_t ix[kFmtMax];
	uint32_t num = 1, sec = 0; int64_t max_score = 0; uint32_t bytes = 0;
	int first_slot = -1; bool qualifies = false;
	if(ok) {
		const uint32_t fl = a.flags[u]; const bool f1 = fl & 1u, f2 = (fl & 2u) != 0;
		if(!uncl) {
			if(f1) { const int64_t L = a.len[0][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
			if(f2) { const int64_t L = a.len[1][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
		}
		Lcg32 rnd; rnd.last = (f1 && f2) ? (a.seedv[0][u] ^ a.seedv[1][u]) : a.seedv[0][u];
		int64_t best = -1, sec64 = -1;                                    // scores are >= 0: -1 plays "invalid"
		for(uint32_t k = 0; k < sz; k++) {
			const uint32_t s = uncl ? 0u : a.recs[r0 + k].score;
			if((int64_t)s > best) { sec64 = best; best = s; } else if((int64_t)s > sec64) sec64 = s;
			sc[k] = s; ix[k] = (uint8_t)k;
		}
		sec = sec64 < 0 ? 0u : (uint32_t)sec64;
		num = sz < a.khits ? sz : a.khits;
		if(sz > 1) {
			// descending by (score, original position): std::sort of pairs followed by reverse
			for(uint32_t i = 1; i < sz; i++) {
				const uint32_t s = sc[i]; const uint8_t x = ix[i]; uint32_t j = i;
				while(j > 0 && (sc[j - 1] < s || (sc[j - 1] == s && ix[j - 1] < x))) { sc[j] = sc[j - 1]; ix[j] = ix[j - 1]; j--; }
				sc[j] = s; ix[j] = x;
			}
			uint32_t streak = 0;
			for(uint32_t k = 1; k <= sz; k++) {
				if(k < sz && sc[k] == sc[k - 1]) { if(streak == 0) streak = 1; streak++; }
				else {
					if(streak > 1) {        // shufflePortion(k - streak, streak)
						const uint32_t begin = k - streak; uint32_t left = streak;
						for(uint32_t i = begin; i < begin + streak - 1; i++) {
							const uint32_t r = rnd.next() % left;
							if(r > 0) { const uint32_t ts = sc[i]; sc[i] = sc[i + r]; sc[i + r] = ts; const uint8_t tx = ix[i]; ix[i] = ix[i + r]; ix[i + r] = tx; }
							left--;
						}
					}
					streak = 0;
				}
			}
			for(uint32_t k = 0; k + 1 < num; k++) if(sc[k] != sc[k + 1]) { num = k + 1; break; }
		}
		ColRow row; unit_row(a, u, row); row.sec = sec; row.num = num;
		uint64_t tie[kFmtMax];
		for(uint32_t k = 0; k < num; k++) {
			if(!uncl) a.sel[r0 + k] = ix[k];
			rec_row(a, uncl, a.recs + r0 + ix[k], row);
			const uint64_t taxid = row.taxid; const uint32_t score = (uint32_t)row.score;
			ColCount cnt; emit_row(cnt, a.cols, a.n_cols, row);
			bytes += (uint32_t)cnt.n;
			const int slot = find_u64(a.tb.sp_taxid, a.tb.n_sp, taxid);
			if(slot < 0) atomicOr(a.tscal, (unsigned long long)TX_FMT_OVERFLOW);   // unknown taxid: let the host path count it
			if(k == 0) { first_slot = slot; qualifies = (int64_t)score >= max_score; }
			else if(slot >= 0) { atomicAdd(a.sp + slot, 1ull); }
			tie[k] = taxid;
		}
		if(qualifies && num > 1) {
			for(uint32_t i = 1; i < num; i++) { const uint64_t t = tie[i]; uint32_t j = i; while(j > 0 && tie[j - 1] > t) { tie[j] = tie[j - 1]; j--; } tie[j] = t; }
			const unsigned long long pos = atomicAdd(a.tscal + 2, 1ull);
			if(pos < a.multi_cap) { unsigned long long* mr = a.multi + pos * a.multi_stride; mr[0] = num; for(uint32_t i = 0; i < num; i++) mr[1 + i] = tie[i]; }
		}
		a.row_bytes[u] = bytes; a.num[u] = (uint8_t)num; a.sec[u] = sec;
	}
	// first row of every unit: warp-aggregated counters (dominant taxa would serialise per-lane atomics)
	const int key = ok ? first_slot : -1;
	const uint32_t peers = __match_any_sync(0xffffffffu, key);
	if(key >= 0) {
		const uint32_t uniq = __popc(__ballot_sync(peers, num == 1) & peers);
		const uint32_t obs = __popc(__ballot_sync(peers, num == 1 && qualifies) & peers);
		if((uint32_t)(__ffs(peers) - 1) == (threadIdx.x & 31u)) {
			atomicAdd(a.sp + key, (unsigned long long)__popc(peers));
			if(uniq) atomicAdd(a.sp + a.tb.n_sp + key, (unsigned long long)uniq);
			if(obs) atomicAdd(a.sp + 2ull * a.tb.n_sp + key, (unsigned long long)obs);
		}
	}
}

static const int kFmtShBytes = 16 * 1024;      // 128 units x ~60-byte rows fit with room to spare; 12 CTAs per SM stay resident
__global__ void __launch_bounds__(128, 8) k_fmt_write(const FmtArgs a) {
	__shared__ char sh[kFmtShBytes];
	if(span_rejected(a)) return;
	const uint32_t u0 = blockIdx.x * 128, u1 = min(u0 + 128u, a.n_units);
	const uint64_t base = a.txt_off[u0], end = a.txt_off[u1], span = end - base;
	if(a.txt_off[a.n_units] > a.out_cap) return;             // host grows the buffer and relaunches
	if(span > (uint64_t)kFmtShBytes) {
		// long rows (sequence / quality columns, long names): warp per unit, straight to global memory
		const uint32_t lane = threadIdx.x & 31, w0 = u0 + (threadIdx.x & ~31u), w1 = min(w0 + 32u, u1);
		for(uint32_t u = w0; u < w1; u++) {
			if(!a.row_bytes[u]) continue;
			const uint32_t r0 = a.rec_off[u], r1 = a.rec_off[u + 1];
			const bool uncl = r0 == r1;
			ColRow row; unit_row(a, u, row); row.sec = a.sec[u]; row.num = a.num[u];
			ColWarpWriter w; w.p = a.out + a.txt_off[u]; w.lane = lane;
			for(uint32_t k = 0; k < row.num; k++) {
				rec_row(a, uncl, uncl ? a.recs : a.recs + r0 + a.sel[r0 + k], row);
				emit_row(w, a.cols, a.n_cols, row);
			}
		}
		return;
	}
	const uint32_t u = u0 + threadIdx.x;
	if(u < u1 && a.row_bytes[u]) {
		const uint32_t r0 = a.rec_off[u], r1 = a.rec_off[u + 1];
		const bool uncl = r0 == r1;
		ColRow row; unit_row(a, u, row); row.sec = a.sec[u]; row.num = a.num[u];
		ColWriter w; w.p = sh + (a.txt_off[u] - base);
		for(uint32_t k = 0; k < row.num; k++) {
			rec_row(a, uncl, uncl ? a.recs : a.recs + r0 + a.sel[r0 + k], row);
			emit_row(w, a.cols, a.n_cols, row);
		}
	}
	__syncthreads();
	for(uint64_t i = threadIdx.x; i < span; i += 128) a.out[base + i] = sh[i];
}
__global__ void k_sp_commit(const unsigned long long* slot_sp, unsigned long long* total, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) { const unsigned long long v = slot_sp[i]; if(v) atomicAdd(total + i, v); }
}

// ------------------------------------------------------------------------------ host glue
struct TextSlot {
	DBuf<uint8_t> d_text[2]; HBuf<uint8_t> h_text[2];
	DBuf<uint32_t> nl[2]; DBuf<uint32_t> tile_cnt[2]; DBuf<uint64_t> tile_off[2]; DBuf<uint64_t> tbsum;
	DBuf<uint32_t> seedv[2], name_off, name_len, id_len, seq_off[2], qual_off[2];
	DBuf<uint32_t> row_bytes, sec; DBuf<uint64_t> txt_off; DBuf<uint8_t> sel, num;
	DBuf<char> d_tsv; HBuf<char> h_tsv; DBuf<unsigned long long> multi; HBuf<unsigned long long> h_multi;
	DBuf<unsigned long long> sp;
	DBuf<unsigned long long> tscal; HBuf<unsigned long long> h_tscal;    // [0] status [1] maxlen [2] n_multi [3] maxlen of mates up to kLongUnitLen [4],[5] line totals [6] tsv bytes
	uint64_t n_rec = 0; int n_mates = 1; cfb_text_opts opt; uint64_t bytes[2] = {0, 0}; bool pending = false;
	NCeil nceil;                    // the context's N ceiling when the span was submitted (re-runs of the span keep it)
	Quals quals;                    // the context's quality encoding when the span was submitted (the same)
	DBuf<uint8_t> qconv[2];         // k_tok_quals' phred33 qualities (spans in another encoding only)
	bool convert() const { return !opt.fasta && !quals.is_default(); }
	uint64_t spec_tsv = 0, spec_multi = 0;      // bytes / tie-set records already copied home behind the kernels
	DBuf<uint8_t> d_cols; std::vector<uint8_t> cols;      // column list of the span in flight (device copy of `cols`)
};
struct TextCtx {
	bool ready = false, names_ready = false;
	DBuf<uint64_t> nd_taxid; DBuf<uint8_t> nd_info; DBuf<uint32_t> sn_off; DBuf<char> sn_blob; DBuf<uint8_t> rk_off; DBuf<char> rk_blob;
	DBuf<uint64_t> nm_taxid; DBuf<uint32_t> nm_off; DBuf<char> nm_blob;      // taxon names, uploaded when a list prints taxName
	std::vector<uint8_t> cols;      // column list of later spans (cfb_ctx_set_columns)
	TextCtx() { ColList l; std::string e; l.parse(kDefaultCols, e); cols = l.fields; }
	FmtTables tb;       // the per-taxon counter space (sp_taxid) and its totals live in the context (CountsCtx)
	uint32_t maxlen_hint = 128;
	double tsv_ratio = 64.0, multi_ratio = 0.05;     // bytes / tie sets per unit seen so far (size the speculative D2H)
	TextSlot slots[kSlots - 1];
};

static int text_init(cfb_ctx* c) {
	if(!c->text) c->text.reset(new TextCtx());
	TextCtx& t = *c->text;
	if(t.ready) return CFB_OK;
	const HostIndex& h = c->ix->h;
	std::vector<uint64_t> nt(h.nodes.size()); std::vector<uint8_t> ni(h.nodes.size());
	for(size_t i = 0; i < h.nodes.size(); i++) { nt[i] = h.nodes[i].taxid; ni[i] = (uint8_t)((h.nodes[i].rank & 0x7f) | (h.nodes[i].leaf ? 0x80 : 0)); }
	{ int rc = counts_init(c); if(rc) return rc; }
	std::vector<uint32_t> so(h.seq_name.size() + 1, 0); std::string blob;
	for(size_t i = 0; i < h.seq_name.size(); i++) { so[i] = (uint32_t)blob.size(); blob += h.seq_name[i]; }
	so[h.seq_name.size()] = (uint32_t)blob.size();
	if(blob.size() >= (1ull << 32)) return fail(CFB_EINVAL, "sequence name table too large for the text operator");
	std::vector<uint8_t> ro(RANK_MAX + 2, 0); std::string rb;
	for(int r = 0; r < RANK_MAX; r++) { ro[r] = (uint8_t)rb.size(); rb += rank_name(r); }
	ro[RANK_MAX] = (uint8_t)rb.size(); rb += "unclassified"; ro[RANK_MAX + 1] = (uint8_t)rb.size();
	if(rb.size() > 255) return fail(CFB_EINVAL, "rank string table overflow");
	#define UP(buf, vec) do { CK(buf.ensure((vec).size() + 1)); if(!(vec).empty()) CK(cudaMemcpy(buf.p, (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice)); } while(0)
	UP(t.nd_taxid, nt); UP(t.nd_info, ni); UP(t.sn_off, so); UP(t.sn_blob, blob); UP(t.rk_off, ro); UP(t.rk_blob, rb);
	#undef UP
	t.tb.nd_taxid = t.nd_taxid.p; t.tb.nd_info = t.nd_info.p; t.tb.n_nodes = (uint32_t)nt.size();
	t.tb.sp_taxid = c->cnt.d_taxid.p; t.tb.n_sp = c->cnt.n;
	t.tb.sn_off = t.sn_off.p; t.tb.sn_blob = t.sn_blob.p; t.tb.n_seq = (uint32_t)h.seq_name.size();
	t.tb.rk_off = t.rk_off.p; t.tb.rk_blob = t.rk_blob.p;
	t.tb.nm_taxid = nullptr; t.tb.nm_off = nullptr; t.tb.nm_blob = nullptr; t.tb.n_names = 0;
	t.ready = true;
	return CFB_OK;
}

// taxName: the index's name table as an ascending taxid array and one blob, as the sequence names
static int text_names_init(cfb_ctx* c) {
	TextCtx& t = *c->text;
	if(t.names_ready) return CFB_OK;
	const HostIndex& h = c->ix->h;
	std::vector<uint64_t> tx; std::vector<uint32_t> off; std::string blob;
	for(std::map<uint64_t, std::string>::const_iterator it = h.names.begin(); it != h.names.end(); ++it) { tx.push_back(it->first); off.push_back((uint32_t)blob.size()); blob += it->second; }
	off.push_back((uint32_t)blob.size());
	if(blob.size() >= (1ull << 32)) return fail(CFB_EINVAL, "name table too large for the text operator");
	#define UP(buf, vec) do { CK(buf.ensure((vec).size() + 1)); if(!(vec).empty()) CK(cudaMemcpy(buf.p, (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice)); } while(0)
	UP(t.nm_taxid, tx); UP(t.nm_off, off); UP(t.nm_blob, blob);
	#undef UP
	t.tb.nm_taxid = t.nm_taxid.p; t.tb.nm_off = t.nm_off.p; t.tb.nm_blob = t.nm_blob.p; t.tb.n_names = (uint32_t)tx.size();
	t.names_ready = true;
	return CFB_OK;
}

extern "C" int cfb_ctx_set_columns(cfb_ctx* c, const char* cols) {
	if(!c) return fail(CFB_EINVAL, "cfb_ctx_set_columns: bad argument");
	ColList l; std::string err;
	if(!l.parse(cols ? cols : kDefaultCols, err)) return fail(CFB_EINVAL, "%s", err.c_str());
	if(l.fields.size() > (size_t)kTextMaxCols) return fail(CFB_EINVAL, "the text operator prints at most %d columns", kTextMaxCols);
	if(!c->text) c->text.reset(new TextCtx());
	c->text->cols = l.fields;
	return CFB_OK;
}

extern "C" int cfb_ctx_set_n_ceil(cfb_ctx* c, int type, double constant, double coeff, double min, double max) {
	if(!c || type < NCEIL_CONST || type > NCEIL_LOG || constant != constant || coeff != coeff || min != min || max != max)
		return fail(CFB_EINVAL, "cfb_ctx_set_n_ceil: bad argument");
	NCeil& f = c->nceil; f.type = type; f.c = constant; f.l = coeff; f.mn = min; f.mx = max;
	return CFB_OK;
}

extern "C" int cfb_ctx_set_quals(cfb_ctx* c, int solexa, int phred64, int integer) {
	if(!c || (solexa != 0 && solexa != 1) || (phred64 != 0 && phred64 != 1) || (integer != 0 && integer != 1))
		return fail(CFB_EINVAL, "cfb_ctx_set_quals: bad argument");
	c->quals.solexa = solexa != 0; c->quals.phred64 = phred64 != 0; c->quals.integer = integer != 0;
	return CFB_OK;
}
static const uint32_t g_sol_steps = solexa_steps();      // the Solexa -> Phred table, as k_tok_quals holds it

static uint32_t len_class(uint32_t maxlen) { return maxlen <= 128 ? 128u : (maxlen <= 160 ? 160u : (maxlen <= 320 ? 320u : ((maxlen + 1023u) / 1024u) * 1024u)); }

static int text_enqueue_format(cfb_ctx* c, Slot& s, TextSlot& t) {
	TextCtx& tc = *c->text;
	const uint64_t n = t.n_rec;
	const uint32_t ublocks = (uint32_t)((n + 127) / 128);
	const uint64_t scan_blocks = (n + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
	const uint32_t stride = c->prm.khits + 1;
	CK(t.row_bytes.ensure(n)); CK(t.sec.ensure(n)); CK(t.num.ensure(n)); CK(t.txt_off.ensure(n + 1)); CK(t.sel.ensure(s.dense_cap + 1));
	CK(t.multi.ensure(n * stride)); CK(t.sp.ensure(3ull * tc.tb.n_sp));
	if(t.d_tsv.cap == 0) CK(t.d_tsv.ensure(n * 96 + 4096));
	CK(cudaMemsetAsync(t.sp.p, 0, 3ull * tc.tb.n_sp * 8, s.st));
	CK(cudaMemsetAsync(t.tscal.p + 2, 0, 8, s.st));
	FmtArgs fa; fa.tb = tc.tb; fa.text = t.d_text[0].p; fa.name_off = t.name_off.p; fa.id_len = t.id_len.p;
	for(int m = 0; m < 2; m++) { fa.len[m] = s.bv.len[m]; fa.seedv[m] = t.seedv[m].p; }
	fa.flags = s.bv.flags; fa.rec_off = s.rec_off32.p; fa.recs = s.dense.p; fa.n_units = (uint32_t)n; fa.n_mates = t.n_mates; fa.khits = c->prm.khits;
	fa.row_bytes = t.row_bytes.p; fa.txt_off = t.txt_off.p; fa.sel = t.sel.p; fa.num = t.num.p; fa.sec = t.sec.p;
	fa.out = t.d_tsv.p; fa.out_cap = t.d_tsv.cap; fa.sp = t.sp.p; fa.multi = t.multi.p; fa.multi_stride = stride; fa.multi_cap = n;
	fa.tscal = t.tscal.p; fa.maxlen_hint = s.maxlen;
	fa.cols = t.d_cols.p; fa.n_cols = (uint32_t)t.cols.size(); fa.col_mask = col_mask(t.cols.data(), fa.n_cols);
	fa.bases = s.bv.bases;
	for(int m = 0; m < 2; m++) { fa.qtext[m] = t.convert() ? t.qconv[m].p : t.d_text[m].p; fa.off[m] = s.bv.off[m]; fa.qual_off[m] = t.qual_off[m].p; fa.nl[m] = t.nl[m].p; }
	fa.lines_per = t.opt.fasta ? 2 : 4; fa.fasta = t.opt.fasta ? 1 : 0; fa.trim5 = t.opt.trim5; fa.trim3 = t.opt.trim3;
	fa.q_int = t.convert() && t.quals.integer ? 1 : 0;
	k_fmt_plan<<<ublocks, 128, 0, s.st>>>(fa);
	k_scan_sums<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(t.row_bytes.p, n, s.bsum.p);
	k_scan_top<<<1, 1024, 0, s.st>>>(s.bsum.p, scan_blocks, (uint64_t*)(t.tscal.p + 6));
	k_scan_apply<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(t.row_bytes.p, n, s.bsum.p, (const uint64_t*)(t.tscal.p + 6), t.txt_off.p);
	k_fmt_write<<<ublocks, 128, 0, s.st>>>(fa);
	c->launches += 5;
	// rows and tie sets follow the kernels home at the size earlier spans suggest; cfb_text_wait fetches a remainder if any
	t.spec_tsv = std::min<uint64_t>(t.d_tsv.cap, (uint64_t)((double)n * tc.tsv_ratio * 1.05) + 4096);
	t.spec_multi = std::min<uint64_t>(n, (uint64_t)((double)n * tc.multi_ratio * 1.2) + 256);
	CK(t.h_tsv.ensure(t.spec_tsv + 1)); CK(t.h_multi.ensure(t.spec_multi * stride + 1));
	CK(cudaMemcpyAsync(t.h_tsv.p, t.d_tsv.p, t.spec_tsv, cudaMemcpyDeviceToHost, s.st));
	CK(cudaMemcpyAsync(t.h_multi.p, t.multi.p, t.spec_multi * stride * 8, cudaMemcpyDeviceToHost, s.st));
	CK(cudaMemcpyAsync(t.h_tscal.p, t.tscal.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s.st));
	CK(cudaGetLastError());
	return CFB_OK;
}

// tokenise + classify + format of the span already uploaded into t.d_text (re-runnable)
static int text_enqueue_all(cfb_ctx* c, Slot& s, TextSlot& t) {
	TextCtx& tc = *c->text;
	const int nm = t.n_mates; const int L = t.opt.fasta ? 2 : 4;
	const uint64_t n = t.n_rec;
	const uint64_t scan_blocks = (n + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
	CK(cudaMemsetAsync(t.tscal.p, 0, 8 * sizeof(unsigned long long), s.st));
	TextArgs ta; memset(&ta, 0, sizeof ta);
	for(int m = 0; m < nm; m++) {
		const uint32_t tiles = (uint32_t)((t.bytes[m] + kTextTile - 1) / kTextTile);
		const uint64_t tsb = ((uint64_t)tiles + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
		k_nl_count<<<tiles, 256, 0, s.st>>>(t.d_text[m].p, (uint32_t)t.bytes[m], t.tile_cnt[m].p, t.tscal.p);
		k_scan_sums<<<(unsigned)tsb, kScanBlock, 0, s.st>>>(t.tile_cnt[m].p, tiles, t.tbsum.p);
		k_scan_top<<<1, 1024, 0, s.st>>>(t.tbsum.p, tsb, (uint64_t*)(t.tscal.p + 4 + m));
		k_scan_apply<<<(unsigned)tsb, kScanBlock, 0, s.st>>>(t.tile_cnt[m].p, tiles, t.tbsum.p, (const uint64_t*)(t.tscal.p + 4 + m), t.tile_off[m].p);
		k_nl_write<<<tiles, 256, 0, s.st>>>(t.d_text[m].p, (uint32_t)t.bytes[m], t.tile_off[m].p, t.nl[m].p, n * L);
		c->launches += 5;
		ta.text[m] = t.d_text[m].p; ta.nbytes[m] = (uint32_t)t.bytes[m]; ta.nl[m] = t.nl[m].p; ta.nl_total[m] = (const uint64_t*)(t.tscal.p + 4 + m);
		ta.len[m] = s.d_len.p + m * n; ta.off[m] = s.d_off.p + m * (n + 1); ta.seedv[m] = t.seedv[m].p; ta.seq_off[m] = t.seq_off[m].p; ta.qual_off[m] = t.qual_off[m].p;
		ta.qconv[m] = t.convert() ? t.qconv[m].p : nullptr; ta.qtext[m] = ta.qconv[m];
	}
	ta.q_bits = t.convert() ? t.quals.bits() : 0; ta.sol_steps = g_sol_steps;
	ta.n_rec = (uint32_t)n; ta.lines_per = L; ta.n_mates = nm; ta.fasta = t.opt.fasta ? 1 : 0; ta.trim5 = t.opt.trim5; ta.trim3 = t.opt.trim3; ta.seed = t.opt.seed;
	ta.flags = s.d_flags.p; ta.name_off = t.name_off.p; ta.name_len = t.name_len.p; ta.id_len = t.id_len.p; ta.bases = s.d_bases.p; ta.tscal = t.tscal.p;
	ta.maxlen_hint = s.maxlen; ta.keep_long = s.longs.empty() ? 0u : 1u;
	ta.nc_type = t.nceil.type; ta.nc_c = t.nceil.c; ta.nc_l = t.nceil.l; ta.nc_mn = t.nceil.mn; ta.nc_mx = t.nceil.mx;
	s.nceil = t.nceil; s.custom_nceil = !t.nceil.is_default();      // sizes the hit lists for the Ns a passing mate may hold
	k_tok_rec<<<(unsigned)((n * nm + 127) / 128), 128, 0, s.st>>>(ta); c->launches++;
	if(t.convert()) { k_tok_quals<<<(unsigned)((n + 3) / 4), 128, 0, s.st>>>(ta); c->launches++; }
	for(int m = 0; m < nm; m++) {
		k_scan_sums<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(s.d_len.p + m * n, n, s.bsum.p);
		k_scan_top<<<1, 1024, 0, s.st>>>(s.bsum.p, scan_blocks, (uint64_t*)(t.tscal.p + 7));
		k_scan_apply<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(s.d_len.p + m * n, n, s.bsum.p, (const uint64_t*)(t.tscal.p + 7), s.d_off.p + m * (n + 1));
		c->launches += 3;
	}
	if(t.convert()) k_tok_bases<true><<<(unsigned)((n + 3) / 4), 128, 0, s.st>>>(ta);
	else k_tok_bases<false><<<(unsigned)((n + 3) / 4), 128, 0, s.st>>>(ta);
	c->launches++;
	CK(cudaGetLastError());
	s.cap = 0; s.reran = false;
	int rc = enqueue_kernels(c, s, 0, false); if(rc) return rc;
	return text_enqueue_format(c, s, t);
}

extern "C" int cfb_text_submit(cfb_ctx* c, int slot, const void* text_a, uint64_t bytes_a, const void* text_b, uint64_t bytes_b,
                               uint64_t n_rec, const cfb_text_opts* o) {
	if(!c || !o || !text_a || slot < 0 || slot >= kSlots - 1) return fail(CFB_EINVAL, "cfb_text_submit: bad argument");
	if(c->prm.khits > (uint32_t)kFmtMax) return fail(CFB_EINVAL, "text operator holds at most %d rows per read (-k)", kFmtMax);
	if(bytes_a >= (1ull << 31) || bytes_b >= (1ull << 31) || n_rec >= (1ull << 28)) return fail(CFB_EINVAL, "text span too large");
	if(o->trim5 < 0 || o->trim3 < 0) return fail(CFB_EINVAL, "negative trim");
	if(n_rec && (bytes_a == 0 || (text_b && bytes_b == 0))) return fail(CFB_EINVAL, "empty text span");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[slot];
	if(s.pending) return fail(CFB_EINVAL, "slot %d still has an un-waited batch", slot);
	int rc = text_init(c); if(rc) return rc;
	TextCtx& tc = *c->text; TextSlot& t = tc.slots[slot];
	if(col_mask(tc.cols.data(), (uint32_t)tc.cols.size()) & (1u << COL_TAX_NAME)) { rc = text_names_init(c); if(rc) return rc; }
	if(t.cols != tc.cols) {       // the slot is idle: its formatter kernels finished in the last cfb_text_wait
		CK(t.d_cols.ensure(tc.cols.size()));
		CK(cudaMemcpy(t.d_cols.p, tc.cols.data(), tc.cols.size(), cudaMemcpyHostToDevice));
		t.cols = tc.cols;
	}
	const int nm = text_b ? 2 : 1; const int L = o->fasta ? 2 : 4;
	t.n_rec = n_rec; t.n_mates = nm; t.opt = *o; t.nceil = c->nceil; t.quals = c->quals; t.bytes[0] = bytes_a; t.bytes[1] = text_b ? bytes_b : 0;
	s.n_units = n_rec; s.bv.n_units = (uint32_t)n_rec; s.bv.n_mates = nm; s.longs.clear(); s.win_first = 0;
	if(n_rec == 0) { s.pending = true; t.pending = true; return CFB_OK; }
	CK(t.tscal.ensure(8)); CK(t.h_tscal.ensure(8));
	const void* src[2] = {text_a, text_b};
	const uint64_t n = n_rec;
	const uint64_t scan_blocks = (n + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
	CK(s.bsum.ensure(scan_blocks + 1));
	CK(s.d_len.ensure(n * nm)); CK(s.d_off.ensure((n + 1) * nm)); CK(s.d_flags.ensure(n)); CK(s.d_bases.ensure(bytes_a + t.bytes[1] + 16));
	CK(t.name_off.ensure(n)); CK(t.name_len.ensure(n)); CK(t.id_len.ensure(n));
	uint64_t max_tsb = 1;
	for(int m = 0; m < nm; m++) {
		CK(t.d_text[m].ensure(t.bytes[m] + 32));
		const void* from = src[m];
		if(!is_pinned(from)) { CK(t.h_text[m].ensure(t.bytes[m])); memcpy(t.h_text[m].p, from, t.bytes[m]); from = t.h_text[m].p; }
		CK(cudaMemcpyAsync(t.d_text[m].p, from, t.bytes[m], cudaMemcpyHostToDevice, s.st));
		const uint32_t tiles = (uint32_t)((t.bytes[m] + kTextTile - 1) / kTextTile);
		CK(t.tile_cnt[m].ensure(tiles)); CK(t.tile_off[m].ensure(tiles + 1)); CK(t.nl[m].ensure(n * L + 1));
		max_tsb = std::max<uint64_t>(max_tsb, ((uint64_t)tiles + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer));
		CK(t.seedv[m].ensure(n)); CK(t.seq_off[m].ensure(n)); CK(t.qual_off[m].ensure(n));
		if(t.convert()) CK(t.qconv[m].ensure(t.bytes[m] + 32));
	}
	CK(t.tbsum.ensure(max_tsb + 1));
	s.bv.bases = s.d_bases.p; s.bv.flags = s.d_flags.p;
	for(int m = 0; m < 2; m++) { s.bv.off[m] = m < nm ? s.d_off.p + m * (n + 1) : nullptr; s.bv.len[m] = m < nm ? s.d_len.p + m * n : nullptr; }
	s.n_bases = bytes_a + t.bytes[1];
	if(o->maxlen_hint) tc.maxlen_hint = std::max(tc.maxlen_hint, len_class(o->maxlen_hint));
	s.maxlen = tc.maxlen_hint; s.want_host = false; s.is_text = true;
	rc = text_enqueue_all(c, s, t); if(rc) return rc;
	s.pending = true; t.pending = true;
	return CFB_OK;
}

extern "C" int cfb_text_wait(cfb_ctx* c, int slot, int discard, cfb_text_result* out) {
	if(!c || !out || slot < 0 || slot >= kSlots - 1 || !c->text) return fail(CFB_EINVAL, "cfb_text_wait: bad argument");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[slot]; TextCtx& tc = *c->text; TextSlot& t = tc.slots[slot];
	if(!s.pending || !t.pending) return fail(CFB_EINVAL, "slot %d has no submitted text span", slot);
	s.pending = false; t.pending = false;
	memset(out, 0, sizeof *out);
	out->n_units = t.n_rec; out->multi_stride = c->prm.khits + 1;
	if(t.n_rec == 0) return CFB_OK;
	for(int attempt = 0; attempt < 8; attempt++) {
		cfb_result r;
		int rc = finish_batch(c, s, false, false, &r); if(rc) return rc;     // syncs; re-runs classification stages that overflowed
		const unsigned st = (unsigned)t.h_tscal.p[0];
		if(st & (TX_IRREGULAR | TX_LINECOUNT)) { out->irregular = 1; return CFB_OK; }
		const uint32_t maxlen = (uint32_t)t.h_tscal.p[3];
		out->maxlen = (uint32_t)t.h_tscal.p[1];
		if(maxlen > s.maxlen) {          // longer reads than the buffers were sized for: redo the span in a wider class
			tc.maxlen_hint = std::max(tc.maxlen_hint, len_class(maxlen)); s.maxlen = tc.maxlen_hint;
			rc = text_enqueue_all(c, s, t); if(rc) return rc;
			continue;
		}
		if(out->maxlen > kLongUnitLen && s.longs.empty()) {     // long records: tokenise again with their flags, and classify them with the long-unit kernels
			const uint64_t n = t.n_rec; const int nm = t.n_mates;
			std::vector<uint32_t> lens(n * nm);
			CK(cudaMemcpy(lens.data(), s.d_len.p, n * nm * sizeof(uint32_t), cudaMemcpyDeviceToHost));
			const uint32_t* L[2] = {lens.data(), nm == 2 ? lens.data() + n : nullptr};
			collect_longs(s, n, nm, L, nullptr);
			rc = text_enqueue_all(c, s, t); if(rc) return rc;
			continue;
		}
		// the formatter ran against the first classification pass; redo it if finish_batch had to repeat stages
		if(s.reran) { s.reran = false; rc = text_enqueue_format(c, s, t); if(rc) return rc; continue; }
		if(st & TX_FMT_OVERFLOW) { out->irregular = 1; return CFB_OK; }
		const uint64_t tsv = t.h_tscal.p[6];
		if(tsv > t.d_tsv.cap) { CK(t.d_tsv.ensure(tsv + tsv / 8)); rc = text_enqueue_format(c, s, t); if(rc) return rc; continue; }
		const uint64_t n_multi = t.h_tscal.p[2];
		tc.tsv_ratio = std::max(tc.tsv_ratio * 0.98, (double)tsv / (double)t.n_rec);
		tc.multi_ratio = std::max(tc.multi_ratio * 0.98, (double)n_multi / (double)t.n_rec);
		bool more = false;
		if(tsv > t.spec_tsv) {
			if(tsv + 1 > t.h_tsv.cap) { CK(t.h_tsv.ensure(tsv + 1)); CK(cudaMemcpyAsync(t.h_tsv.p, t.d_tsv.p, tsv, cudaMemcpyDeviceToHost, s.st)); }
			else CK(cudaMemcpyAsync(t.h_tsv.p + t.spec_tsv, t.d_tsv.p + t.spec_tsv, tsv - t.spec_tsv, cudaMemcpyDeviceToHost, s.st));
			more = true;
		}
		if(n_multi > t.spec_multi) {
			CK(t.h_multi.ensure(n_multi * out->multi_stride + 1));
			CK(cudaMemcpyAsync(t.h_multi.p, t.multi.p, n_multi * out->multi_stride * 8, cudaMemcpyDeviceToHost, s.st));
			more = true;
		}
		if(!discard) { const uint32_t nsp3 = 3 * tc.tb.n_sp; k_sp_commit<<<(nsp3 + 255) / 256, 256, 0, s.st>>>(t.sp.p, c->cnt.total.p, nsp3); c->launches++; c->cnt.reduced = false;
			CK(cudaEventRecord(s.ev[5], s.st)); s.commit_pending = true; }
		if(more) CK(cudaStreamSynchronize(s.st));
		out->tsv = t.h_tsv.p; out->tsv_bytes = tsv; out->multi = (const uint64_t*)t.h_multi.p; out->n_multi = n_multi;
		return CFB_OK;
	}
	return fail(CFB_ECUDA, "text operator did not converge");
}

extern "C" int cfb_text_species(cfb_ctx* c, uint64_t* taxid, uint64_t* n_reads, uint64_t* n_unique, uint64_t* n_obs1, uint64_t cap, uint64_t* n) {
	return cfb_counts_read(c, 0, taxid, n_reads, n_unique, n_obs1, cap, n);
}
