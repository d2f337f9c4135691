// tests/native/bunzip2_host.cpp -- TEST ONLY.  Compiles the device decompressor's per-block stages
// (centrifuge_b200/csrc/cf_bzip2.h) for the host, so that tests/test_bunzip2_host.py can check them against Python's bz2
// without a GPU.  The inverse BWT here is libbz2's sequential walk, written out only to check decode_block and the
// RLE1 and CRC stages: this is not a CPU fallback, and nothing in the product links or loads this file.
#include <vector>
#include "../../centrifuge_b200/csrc/cf_bzip2.h"

extern "C" {

// res: {status, n, orig_ptr, crc, end_bit, n_groups, n_selectors}; L must hold BLOCK_MAX bytes
void bzh_decode_block(const uint8_t* in, uint64_t n, uint64_t start, uint8_t* L, int64_t* res) {
	static cbz::Work w;
	cbz::BlockResult r;
	cbz::decode_block(in, n, start, cbz::BLOCK_MAX, L, w, r);
	res[0] = r.status; res[1] = r.n; res[2] = r.orig_ptr; res[3] = r.crc; res[4] = (int64_t)r.end_bit; res[5] = r.n_groups; res[6] = r.n_selectors;
}

// the 48-bit magic at every bit offset in [from, to): block magics as b, end-of-stream magics as -1 - b
uint64_t bzh_scan(const uint8_t* in, uint64_t n, uint64_t from, uint64_t to, int64_t* out, uint64_t cap) {
	uint64_t k = 0;
	for(uint64_t b = from; b < to; b++) {
		const uint64_t m = cbz::read48(in, n, b);
		if(m == cbz::MAGIC_BLOCK || m == cbz::MAGIC_EOS) { if(k < cap) out[k] = m == cbz::MAGIC_BLOCK ? (int64_t)b : -1 - (int64_t)b; k++; }
	}
	return k;
}

// L of n bytes -> the block's output (at most cap bytes; returns its length, or -1 for a block ending in a run without
// its count, -2 when cap is too small) and its CRC in *crc.  seg > 0: RLE1 and CRC run in segments of seg bytes from the
// start states the device chains (rle1_step from each of the five states), combined with crc_extend.
int64_t bzh_block_output(const uint8_t* L, uint32_t n, uint32_t orig_ptr, uint32_t seg, uint8_t* out, uint64_t cap, uint32_t* crc) {
	std::vector<uint32_t> cnt(256, 0), tt(n);
	for(uint32_t i = 0; i < n; i++) cnt[L[i]]++;
	uint32_t s = 0;
	for(int c = 0; c < 256; c++) { const uint32_t v = cnt[c]; cnt[c] = s; s += v; }
	for(uint32_t i = 0; i < n; i++) tt[cnt[L[i]]++] = i << 8 | L[i];
	std::vector<uint8_t> D(n);
	uint32_t p = tt[orig_ptr] >> 8;
	for(uint32_t k = 0; k < n; k++) { const uint32_t e = tt[p]; D[k] = (uint8_t)L[p]; p = e >> 8; }
	uint32_t tab[256];
	for(uint32_t i = 0; i < 256; i++) tab[i] = cbz::crc_table_entry(i);
	if(!seg) seg = n;
	uint64_t o = 0; uint32_t reg_all = 0xFFFFFFFFu; int r = 0;
	for(uint32_t lo = 0; lo < n; lo += seg) {
		const uint32_t hi = lo + seg < n ? lo + seg : n;
		// the segment from every start state, as k_bz_rle_count does; the chained state picks one
		int rs[5] = {0, 1, 2, 3, 4}; uint64_t len[5] = {0, 0, 0, 0, 0};
		uint8_t prev = lo ? D[lo - 1] : 0;
		for(uint32_t i = lo; i < hi; i++) { for(int q = 0; q < 5; q++) len[q] += cbz::rle1_step(rs[q], D[i], prev); prev = D[i]; }
		uint32_t reg = 0; const uint64_t o0 = o;
		prev = lo ? D[lo - 1] : 0;
		int rr = r;
		for(uint32_t i = lo; i < hi; i++) {
			const uint8_t x = D[i];
			const int was = rr;
			const uint32_t k = cbz::rle1_step(rr, x, prev);
			const uint8_t c = was == 4 ? prev : x;
			for(uint32_t j = 0; j < k; j++) { if(o >= cap) return -2; out[o++] = c; reg = (reg << 8) ^ tab[(reg >> 24) ^ c]; }
			prev = x;
		}
		if(rr != rs[r] || o - o0 != len[r]) return -3;
		r = rr;
		reg_all = cbz::crc_extend(reg_all, reg, o - o0);
	}
	if(r == 4) return -1;
	*crc = ~reg_all;
	return (int64_t)o;
}

uint32_t bzh_crc(const uint8_t* p, uint64_t n) {
	uint32_t c = 0xFFFFFFFFu;
	for(uint64_t i = 0; i < n; i++) c = (c << 8) ^ cbz::crc_table_entry((c >> 24) ^ p[i]);
	return ~c;
}

}
