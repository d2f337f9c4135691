// cf_bzip2.h -- bzip2 block decoding stages as __host__ __device__ functions.
//
// The device decompressor (cf_bunzip2.cu) runs these per thread: k_bz_decode turns one candidate block into its BWT
// column L with decode_block, k_bz_rle_count / k_bz_expand undo the final run-length stage segment by segment with
// rle1_step, and k_bz_crc combines the segments' CRCs with crc_mul / crc_xpow8.  tests/native/bunzip2_host.cpp compiles
// the same code for the host and checks it against Python's bz2.  Nothing in the product runs them on the CPU.
//
// Every read is bounded by the input length and every loop by the input or by the largest block the format allows:
// a false block start or a malformed stream yields a negative status, never an out-of-bounds access.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define CBZ_HD __host__ __device__ __forceinline__
#else
#define CBZ_HD inline
#endif

namespace cbz {

constexpr uint64_t NONE = ~0ull;
constexpr uint32_t BLOCK_MAX = 900000;            // level 9: the largest BWT block
constexpr int MAX_GROUPS = 6, MAX_ALPHA = 258, MAX_SELECTORS = 18002, MAX_LEN = 20, GROUP_SIZE = 50;
// +1/-1 steps of one code length: an encoder writes |difference| <= 19 of them.  A block that pads more is rejected
// (libbz2 would read on), so every block this decoder accepts fits in MAX_BLOCK_BITS.
constexpr int MAX_LEN_STEPS = 40;
constexpr uint64_t MAX_BLOCK_BITS = 48 + 32 + 1 + 24 + 16 + 16 * 16          // magic, CRC, randomised, origPtr, symbol map
                                  + 3 + 15 + 32767ull * MAX_GROUPS           // nGroups, nSelectors, unary selectors
                                  + MAX_GROUPS * (5 + MAX_ALPHA * (2ull * MAX_LEN_STEPS + 1))      // code lengths
                                  + (uint64_t)MAX_SELECTORS * GROUP_SIZE * MAX_LEN;                // symbols
constexpr uint64_t MAGIC_BLOCK = 0x314159265359ull, MAGIC_EOS = 0x177245385090ull;
constexpr uint32_t CRC_POLY = 0x04C11DB7u;

enum : int {
	OK = 0,
	E_INPUT = -1,        // ran past the end of the input
	E_MAGIC = -2,        // no block magic at the start
	E_RANDOMISED = -3,   // the obsolete randomised bit is set
	E_MAP = -4,          // no byte value in use
	E_GROUPS = -5,       // nGroups outside 2..6
	E_SELECTORS = -6,    // no selectors, a selector >= nGroups, or the data runs past the last selector
	E_LENGTHS = -7,      // a code length outside 1..20, or more than MAX_LEN_STEPS steps to one
	E_CODE = -8,         // a bit pattern that is no code of the group's table
	E_SIZE = -9,         // the block is longer than its level allows
	E_ORIGPTR = -10,     // origPtr outside the block
	E_RLE = -11,         // the block ends after four equal bytes, without their count
};

CBZ_HD const char* status_text(int s) {
	switch(s) {
	case E_INPUT: return "unexpected end of the compressed stream";
	case E_MAGIC: return "bad block header magic";
	case E_RANDOMISED: return "randomised block (obsolete bzip2 format before 0.9.5, not supported)";
	case E_MAP: return "invalid symbol map (no byte in use)";
	case E_GROUPS: return "invalid number of Huffman groups";
	case E_SELECTORS: return "invalid selectors";
	case E_LENGTHS: return "invalid code lengths";
	case E_CODE: return "invalid Huffman code";
	case E_SIZE: return "block longer than its level allows";
	case E_ORIGPTR: return "origPtr out of range";
	case E_RLE: return "invalid run-length data";
	default: return "ok";
	}
}

// MSB-first bit reader over in[0, n); bytes past the end read as zero and over() tells that they were used
struct Bits {
	const uint8_t* p; uint64_t n, next; uint64_t buf; int cnt;
	CBZ_HD void init(const uint8_t* p_, uint64_t n_, uint64_t bitpos) {
		p = p_; n = n_; next = bitpos >> 3; buf = 0; cnt = 0;
		refill(); drop((int)(bitpos & 7));
	}
	CBZ_HD void refill() {
		while(cnt <= 56) { const uint64_t b = next < n ? p[next] : 0; buf |= b << (56 - cnt); next++; cnt += 8; }
	}
	CBZ_HD uint32_t peek(int k) const { return (uint32_t)(buf >> (64 - k)); }          // 1 <= k <= 32
	CBZ_HD void drop(int k) { buf <<= k; cnt -= k; }
	CBZ_HD uint32_t get(int k) { const uint32_t v = peek(k); drop(k); return v; }      // k <= cnt: callers refill first
	CBZ_HD uint64_t pos() const { return next * 8 - (uint64_t)cnt; }
	CBZ_HD bool over() const { return pos() > n * 8; }
};

// the 48 bits at bit b of in[0, n) (zeros past the end)
CBZ_HD uint64_t read48(const uint8_t* in, uint64_t n, uint64_t b) {
	Bits r; r.init(in, n, b);
	return (uint64_t)r.peek(24) << 24 | (uint64_t)(uint32_t)((r.buf >> 16) & 0xffffff);
}

// per-decoder tables: shared memory on the device (about 6 KB)
struct Work {
	int32_t limit[MAX_GROUPS][MAX_LEN + 1];
	int32_t base[MAX_GROUPS][MAX_LEN + 2];
	uint16_t perm[MAX_GROUPS][MAX_ALPHA];
	uint16_t nperm[MAX_GROUPS];
	uint8_t minlen[MAX_GROUPS];
	uint8_t len[MAX_ALPHA];
	uint8_t seq2byte[256];
	uint8_t mtf[256];
	uint32_t hist[256];
};

struct BlockResult {
	int32_t status;
	uint32_t n;              // BWT bytes (length of L)
	uint32_t orig_ptr;
	uint32_t crc;            // the block CRC stored in its header
	uint64_t end_bit;        // first bit after the end-of-block symbol
	uint32_t n_groups, n_selectors;
};

// canonical decode tables of one group (codes in order of length, then symbol), libbz2's limit/base/perm form
CBZ_HD void build_tables(Work& w, int t, int alpha) {
	int mn = 32, mx = 0;
	for(int i = 0; i < alpha; i++) { mn = w.len[i] < mn ? w.len[i] : mn; mx = w.len[i] > mx ? w.len[i] : mx; }
	int pp = 0;
	for(int l = mn; l <= mx; l++) for(int s = 0; s < alpha; s++) if(w.len[s] == l) w.perm[t][pp++] = (uint16_t)s;
	w.nperm[t] = (uint16_t)pp;
	int32_t* base = w.base[t]; int32_t* limit = w.limit[t];
	for(int i = 0; i < MAX_LEN + 2; i++) base[i] = 0;
	for(int s = 0; s < alpha; s++) base[w.len[s] + 1]++;
	for(int i = 1; i < MAX_LEN + 2; i++) base[i] += base[i - 1];
	for(int i = 0; i <= MAX_LEN; i++) limit[i] = -1;
	int32_t vec = 0;
	for(int l = mn; l <= mx; l++) { vec += base[l + 1] - base[l]; limit[l] = vec - 1; vec <<= 1; }
	for(int l = mn + 1; l <= mx; l++) base[l] = ((limit[l - 1] + 1) << 1) - base[l];
	w.minlen[t] = (uint8_t)mn;
}

// one symbol of group t; < 0 on a bit pattern that is no code
CBZ_HD int decode_sym(Bits& b, const Work& w, int t) {
	int zn = w.minlen[t];
	const uint32_t bits = b.peek(MAX_LEN);
	int32_t zvec = (int32_t)(bits >> (MAX_LEN - zn));
	while(zvec > w.limit[t][zn]) {
		if(++zn > MAX_LEN) return E_CODE;
		zvec = (int32_t)(bits >> (MAX_LEN - zn));
	}
	const int32_t idx = zvec - w.base[t][zn];
	if(idx < 0 || idx >= (int32_t)w.nperm[t]) return E_CODE;
	b.drop(zn);
	return w.perm[t][idx];
}

// Decode the block whose magic starts at bit `start` of in[0, n) into its BWT column L[0, r.n) (at most max_n bytes)
// and w.hist (count of every byte value in L).  Selectors are read twice (once to skip them, once while decoding
// the symbols) so that no selector array is needed.
CBZ_HD void decode_block(const uint8_t* in, uint64_t n, uint64_t start, uint32_t max_n, uint8_t* L, Work& w, BlockResult& r) {
	r.status = OK; r.n = 0; r.orig_ptr = 0; r.crc = 0; r.end_bit = NONE; r.n_groups = 0; r.n_selectors = 0;
	Bits b; b.init(in, n, start);
#define CBZ_FAIL(e) do { r.status = b.over() ? E_INPUT : (e); return; } while(0)
	const uint64_t magic = (uint64_t)b.get(24) << 24 | b.get(24);
	if(magic != MAGIC_BLOCK) CBZ_FAIL(E_MAGIC);
	b.refill();
	r.crc = b.get(16) << 16; r.crc |= b.get(16);
	if(b.get(1)) CBZ_FAIL(E_RANDOMISED);
	r.orig_ptr = b.get(24);
	b.refill();
	const uint32_t in_use16 = b.get(16);
	int n_in_use = 0;
	for(int i = 0; i < 16; i++) {
		if(!(in_use16 >> (15 - i) & 1)) continue;
		b.refill();
		const uint32_t m = b.get(16);
		for(int j = 0; j < 16; j++) if(m >> (15 - j) & 1) w.seq2byte[n_in_use++] = (uint8_t)(i * 16 + j);
	}
	if(b.over()) CBZ_FAIL(E_INPUT);
	if(n_in_use == 0) CBZ_FAIL(E_MAP);
	const int alpha = n_in_use + 2;
	b.refill();
	const int n_groups = (int)b.get(3);
	if(n_groups < 2 || n_groups > MAX_GROUPS) CBZ_FAIL(E_GROUPS);
	const int n_sel = (int)b.get(15);
	if(n_sel < 1) CBZ_FAIL(E_SELECTORS);
	r.n_groups = (uint32_t)n_groups; r.n_selectors = (uint32_t)n_sel;
	const uint64_t sel_bit = b.pos();
	for(int i = 0; i < n_sel; i++) {              // skip (and check) the selectors; those past MAX_SELECTORS are ignored
		b.refill();
		int j = 0;
		while(b.get(1)) { if(++j >= n_groups) CBZ_FAIL(E_SELECTORS); }
		if(b.over()) CBZ_FAIL(E_INPUT);
	}
	const int sel_used = n_sel < MAX_SELECTORS ? n_sel : MAX_SELECTORS;
	for(int t = 0; t < n_groups; t++) {
		b.refill();
		int curr = (int)b.get(5);
		for(int s = 0; s < alpha; s++) {
			for(int steps = 0;; steps++) {
				if(curr < 1 || curr > MAX_LEN || steps > MAX_LEN_STEPS) CBZ_FAIL(E_LENGTHS);
				if(b.cnt < 8) b.refill();
				if(!b.get(1)) break;
				curr += b.get(1) ? -1 : 1;
			}
			w.len[s] = (uint8_t)curr;
		}
		if(b.over()) CBZ_FAIL(E_INPUT);
		build_tables(w, t, alpha);
	}
	// symbols: groups of 50, RUNA/RUNB runs of the front byte, MTF indices, EOB
	for(int i = 0; i < 256; i++) { w.mtf[i] = (uint8_t)i; w.hist[i] = 0; }
	uint8_t sel_mtf[MAX_GROUPS];
	for(int t = 0; t < MAX_GROUPS; t++) sel_mtf[t] = (uint8_t)t;
	Bits sb; sb.init(in, n, sel_bit);
	const int eob = n_in_use + 1;
	uint32_t nb = 0;
	int group_no = -1, group_pos = 0, gsel = 0;
	uint32_t run = 0, run_w = 1;
	for(;;) {
		if(group_pos == 0) {
			if(++group_no >= sel_used) CBZ_FAIL(E_SELECTORS);
			group_pos = GROUP_SIZE;
			sb.refill();
			int j = 0;
			while(sb.get(1)) j++;                  // < n_groups: checked by the skip above
			const uint8_t v = sel_mtf[j];
			for(; j > 0; j--) sel_mtf[j] = sel_mtf[j - 1];
			sel_mtf[0] = v; gsel = v;
		}
		group_pos--;
		if(b.cnt < 32) b.refill();
		const int sym = decode_sym(b, w, gsel);
		if(sym < 0) CBZ_FAIL(sym);
		if(b.over()) CBZ_FAIL(E_INPUT);
		if(sym <= 1) {                              // RUNA / RUNB: bijective base-2 digits of a run length
			run += (uint32_t)(sym + 1) * run_w; run_w <<= 1;
			if(run > max_n) CBZ_FAIL(E_SIZE);
			continue;
		}
		if(run) {
			if(nb + run > max_n) CBZ_FAIL(E_SIZE);
			const uint8_t c = w.seq2byte[w.mtf[0]];
			w.hist[c] += run;
			for(uint32_t k = 0; k < run; k++) L[nb + k] = c;
			nb += run; run = 0; run_w = 1;
		}
		if(sym == eob) break;
		if(nb >= max_n) CBZ_FAIL(E_SIZE);
		int idx = sym - 1;
		const uint8_t v = w.mtf[idx];
		for(; idx > 0; idx--) w.mtf[idx] = w.mtf[idx - 1];
		w.mtf[0] = v;
		const uint8_t c = w.seq2byte[v];
		w.hist[c]++;
		L[nb++] = c;
	}
	if(r.orig_ptr >= nb) CBZ_FAIL(E_ORIGPTR);
	r.n = nb; r.end_bit = b.pos();
#undef CBZ_FAIL
}

// ---- RLE1 (the first run-length stage of the encoder), undone segment by segment.
// The state before a byte is the number of equal bytes just seen, 0..4 (4: this byte is a count); whenever it is
// above 0 the repeated byte is the previous byte, so a segment's behaviour depends only on its start state.
// One step: returns the bytes the input byte x stands for (a count byte: x copies of prev; otherwise x itself once).
CBZ_HD uint32_t rle1_step(int& r, uint8_t x, uint8_t prev) {
	if(r == 4) { r = 0; return x; }
	if(r > 0 && x == prev) r++;
	else r = 1;
	return 1;
}

// ---- CRC-32 of bzip2: polynomial 0x04C11DB7, MSB first, init and final xor 0xFFFFFFFF
CBZ_HD uint32_t crc_table_entry(uint32_t i) {
	uint32_t c = i << 24;
	for(int k = 0; k < 8; k++) c = c & 0x80000000u ? (c << 1) ^ CRC_POLY : c << 1;
	return c;
}
// a * b modulo the CRC polynomial (bit k = x^k)
CBZ_HD uint32_t crc_mul(uint32_t a, uint32_t b) {
	uint32_t p = 0;
	for(int i = 31; i >= 0; i--) {
		p = p & 0x80000000u ? (p << 1) ^ CRC_POLY : p << 1;
		if(a >> i & 1) p ^= b;
	}
	return p;
}
// x^(8 n) modulo the CRC polynomial
CBZ_HD uint32_t crc_xpow8(uint64_t n) {
	uint32_t p = 1, sq = 0x100;
	while(n) { if(n & 1) p = crc_mul(p, sq); sq = crc_mul(sq, sq); n >>= 1; }
	return p;
}
// a CRC register `reg` after `len` further bytes whose register from 0 is `piece`
CBZ_HD uint32_t crc_extend(uint32_t reg, uint32_t piece, uint64_t len) { return crc_mul(reg, crc_xpow8(len)) ^ piece; }

}  // namespace cbz
