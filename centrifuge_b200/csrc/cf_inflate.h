// cf_inflate.h -- DEFLATE (RFC 1951) decoding of one chunk of a stream, as __host__ __device__ functions.
//
// The device inflater (cf_gunzip.cu) runs these per thread: k_search tests candidate block starts with
// block_header_plausible, k_decode decodes a chunk with inflate_chunk.  tests/native/gunzip_host.cpp compiles the same
// code for the host and checks it against zlib.  Nothing in the product runs them on the CPU.
//
// A chunk decodes into 16-bit symbols: values < 256 are bytes, 256 + w is byte w of the 32 KB window that precedes
// the chunk (w = 0 is the oldest).  Copies inside the chunk copy symbols, so every marker refers to that window, which
// is resolved later.  Every read is bounded by the input length and every loop by the input or the output capacity:
// a malformed stream yields a negative status, never an out-of-bounds access.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define CFZ_HD __host__ __device__ __forceinline__
#else
#define CFZ_HD inline
#endif

namespace cfz {

constexpr uint64_t NONE = ~0ull;
constexpr int WIN = 32768;
constexpr int LUT_LIT = 10, LUT_DIST = 8, LUT_CL = 7;

enum : int {
	ST_STOP = 1,    // reached a block boundary at or after the stop bit
	ST_END = 2,     // decoded the final block
	ST_FULL = 3,    // the symbol buffer is full: stopped before a symbol (or before a stored block)
	E_INPUT = -1,   // ran past the end of the input
	E_BTYPE = -2,   // reserved block type
	E_STORED = -3,  // stored block length does not match its complement
	E_CODES = -4,   // invalid code lengths: over-subscribed or incomplete code, too many symbols, bad repeat
	E_SYM = -5,     // invalid literal/length or distance code
	E_DIST = -6,    // distance reaches before the start of the output
};

CFZ_HD const char* status_text(int s) {
	switch(s) {
	case E_INPUT: return "unexpected end of the compressed stream";
	case E_BTYPE: return "invalid block type";
	case E_STORED: return "invalid stored block lengths";
	case E_CODES: return "invalid code lengths";
	case E_SYM: return "invalid literal/length or distance code";
	case E_DIST: return "invalid distance too far back";
	default: return "ok";
	}
}

// LSB-first bit reader over in[0, n); bytes past the end read as zero and over() tells that they were used
struct Bits {
	const uint8_t* p; uint64_t n, next; uint64_t buf; int cnt;
	CFZ_HD void init(const uint8_t* p_, uint64_t n_, uint64_t bitpos) {
		p = p_; n = n_; next = bitpos >> 3; buf = 0; cnt = 0;
		refill(); drop((int)(bitpos & 7));
	}
	CFZ_HD void refill() {
		while(cnt <= 56) { const uint64_t b = next < n ? p[next] : 0; buf |= b << cnt; next++; cnt += 8; }
	}
	CFZ_HD uint32_t peek(int k) const { return (uint32_t)(buf & ((1ull << k) - 1)); }
	CFZ_HD void drop(int k) { buf >>= k; cnt -= k; }
	CFZ_HD uint32_t get(int k) { const uint32_t v = peek(k); drop(k); return v; }      // k <= cnt: callers refill first
	CFZ_HD uint64_t pos() const { return next * 8 - (uint64_t)cnt; }
	CFZ_HD bool over() const { return pos() > n * 8; }
};

// canonical Huffman code: a direct table for codes of up to `lutb` bits, the counts and sorted symbols for longer ones
template <int LUTB, int NSYM> struct Huff {
	uint16_t lut[1 << LUTB];       // (symbol << 4) | length, 0 = longer code (or none)
	uint16_t count[16];
	uint16_t sym[NSYM];
};

// returns < 0 when over-subscribed, 0 when complete, > 0 when incomplete; *maxlen = longest length used
template <int LUTB, int NSYM> CFZ_HD int huff_build(Huff<LUTB, NSYM>& h, const uint8_t* len, int n, int* maxlen) {
	uint16_t offs[16];
	for(int l = 0; l < 16; l++) h.count[l] = 0;
	for(int s = 0; s < n; s++) h.count[len[s]]++;
	h.count[0] = 0;
	int left = 1, mx = 0;
	for(int l = 1; l < 16; l++) { left <<= 1; left -= h.count[l]; if(left < 0) return -1; if(h.count[l]) mx = l; }
	*maxlen = mx;
	offs[1] = 0;
	for(int l = 1; l < 15; l++) offs[l + 1] = (uint16_t)(offs[l] + h.count[l]);
	for(int s = 0; s < n; s++) if(len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
	for(int j = 0; j < (1 << LUTB); j++) h.lut[j] = 0;
	uint32_t code = 0; int idx = 0;
	for(int l = 1; l <= LUTB; l++) {
		for(int k = 0; k < h.count[l]; k++, idx++, code++) {
			uint32_t r = 0;
			for(int b = 0; b < l; b++) r |= ((code >> b) & 1u) << (l - 1 - b);
			const uint16_t e = (uint16_t)((h.sym[idx] << 4) | l);
			for(uint32_t j = r; j < (1u << LUTB); j += 1u << l) h.lut[j] = e;
		}
		code <<= 1;
	}
	return left;
}

// next symbol, or -1 for a bit pattern the code does not have; needs 15 bits in the buffer
template <int LUTB, int NSYM> CFZ_HD int huff_decode(const Huff<LUTB, NSYM>& h, Bits& b) {
	const uint32_t e = h.lut[b.peek(LUTB)];
	if(e) { b.drop((int)(e & 15)); return (int)(e >> 4); }
	uint64_t bits = b.buf;
	int code = 0, first = 0, index = 0;
	for(int l = 1; l < 16; l++) {
		code |= (int)(bits & 1); bits >>= 1;
		const int c = h.count[l];
		if(code - c < first) { b.drop(l); return h.sym[index + (code - first)]; }
		index += c; first += c; first <<= 1; code <<= 1;
	}
	return -1;
}

struct Tables {
	Huff<LUT_LIT, 288> lit;
	Huff<LUT_DIST, 32> dist;
	Huff<LUT_CL, 19> cl;
	uint8_t lens[320];
};

// Block header at the reader's position (BFINAL and BTYPE already consumed, type 1 or 2): builds the tables.
// strict: what a block start found by searching must satisfy (complete codes only), else zlib's rules
// (an incomplete literal/length or distance code is allowed only when its longest code has one bit).
CFZ_HD int read_tables(Bits& b, int type, Tables& t, bool strict) {
	int mx;
	if(type == 1) {
		for(int s = 0; s < 288; s++) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
		for(int s = 0; s < 30; s++) t.lens[288 + s] = 5;
		huff_build(t.lit, t.lens, 288, &mx);
		huff_build(t.dist, t.lens + 288, 30, &mx);
		return 0;
	}
	const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	b.refill();
	const int hlit = (int)b.get(5) + 257, hdist = (int)b.get(5) + 1, hclen = (int)b.get(4) + 4;
	if(hlit > 286 || hdist > 30) return E_CODES;
	uint8_t cl[19];
	for(int i = 0; i < 19; i++) cl[i] = 0;
	b.refill();
	for(int i = 0; i < hclen; i++) cl[order[i]] = (uint8_t)b.get(3);
	if(huff_build(t.cl, cl, 19, &mx) != 0) return E_CODES;          // the code-length code must be complete
	const int total = hlit + hdist;
	for(int i = 0; i < total;) {
		if(b.over()) return E_INPUT;
		b.refill();
		const int s = huff_decode(t.cl, b);
		if(s < 0) return E_CODES;
		if(s < 16) { t.lens[i++] = (uint8_t)s; continue; }
		int rep; uint8_t v = 0;
		if(s == 16) { if(i == 0) return E_CODES; v = t.lens[i - 1]; rep = 3 + (int)b.get(2); }
		else if(s == 17) rep = 3 + (int)b.get(3);
		else rep = 11 + (int)b.get(7);
		if(i + rep > total) return E_CODES;
		while(rep--) t.lens[i++] = v;
	}
	if(b.over()) return E_INPUT;
	if(t.lens[256] == 0) return E_CODES;                             // no end-of-block code
	int r = huff_build(t.lit, t.lens, hlit, &mx);
	if(r < 0 || (r > 0 && (strict || mx != 1))) return E_CODES;
	uint8_t* dl = t.lens + hlit;
	r = huff_build(t.dist, dl, hdist, &mx);
	if(r < 0 || (r > 0 && (strict || mx > 1))) return E_CODES;        // all-zero distance lengths (mx = 0): no matches allowed
	return 0;
}

// Could a block start at `bit`?  A non-final stored block (zero padding, LEN = ~NLEN) or a dynamic block with complete
// codes; fixed blocks are not searched for (three bits say too little).  Bounded by the input length.
CFZ_HD bool block_header_plausible(const uint8_t* in, uint64_t n, uint64_t bit, Tables& t) {
	if(bit + 3 > n * 8) return false;
	Bits b; b.init(in, n, bit);
	const uint32_t h = b.get(3);
	if(h == 0) {                                                     // BFINAL 0, stored
		const int pad = b.cnt & 7;
		if(b.peek(pad) != 0) return false;
		b.drop(pad);
		const uint32_t len = b.get(16), nlen = b.get(16);
		return !b.over() && len == (~nlen & 0xffffu) && b.pos() / 8 + len <= n;
	}
	if((h >> 1) != 2) return false;
	return read_tables(b, 2, t, true) == 0 && !b.over();
}

// block_header_plausible, then the whole block: a dynamic block must reach its end-of-block code without running past
// the input, and the header after it must be plausible too (any non-reserved type).  Real streams pass; a false start
// that passes the header check almost never does.
CFZ_HD bool block_start_verified(const uint8_t* in, uint64_t n, uint64_t bit, Tables& t) {
	if(!block_header_plausible(in, n, bit, t)) return false;
	Bits b; b.init(in, n, bit);
	const uint32_t h = b.get(3);
	if(h == 0) return true;                                          // stored: LEN = ~NLEN and zero padding already say enough
	if(read_tables(b, 2, t, true) != 0) return false;
	for(;;) {
		if(b.over()) return true;                                    // the input ends inside the block: nothing contradicts it
		b.refill();
		int s = huff_decode(t.lit, b);
		if(s < 0 || s > 285) return false;
		if(s < 256) continue;
		if(s == 256) break;
		s -= 257;
		b.drop(s < 8 || s == 28 ? 0 : (s >> 2) - 1);
		const int ds = huff_decode(t.dist, b);
		if(ds < 0 || ds >= 30) return false;
		b.drop(ds < 4 ? 0 : (ds >> 1) - 1);
	}
	if(h & 1) return true;                                           // final block
	if(b.pos() + 3 > n * 8) return true;
	return block_header_plausible(in, n, b.pos(), t) || ((b.peek(3) >> 1) == 1);
}

struct ChunkResult {
	uint64_t end_bit, end_hdr;      // where decoding stopped; end_hdr != NONE: inside the Huffman block whose header is there
	uint64_t safe_bit, safe_hdr;    // the last state passed that a decode can resume from, and the symbols produced before it
	uint32_t safe_sym;
	uint32_t n_sym;
	int32_t status;
	int32_t first_type;             // type of the first block decoded (-1: none)
};

// Decode from state (start_bit, start_hdr) until the first block boundary at or after stop_bit, the end of the final
// block, cap symbols, or an error.  start_hdr != NONE resumes inside the Huffman block whose header is at start_hdr.
CFZ_HD void inflate_chunk(const uint8_t* in, uint64_t n, uint64_t start_bit, uint64_t start_hdr, uint64_t stop_bit,
                          uint16_t* out, uint32_t cap, Tables& t, ChunkResult& r) {
	uint32_t ns = 0;
	r.first_type = -1;
	r.safe_bit = start_bit; r.safe_hdr = start_hdr; r.safe_sym = 0;
	Bits b;
	bool resume = start_hdr != NONE;
	b.init(in, n, resume ? start_hdr : start_bit);
	// an error met within a code's reach of the end of the input may be the input being short, not the data being bad
	auto finish = [&](int st, uint64_t eb, uint64_t eh) { r.status = st < 0 && b.pos() + 64 > n * 8 ? E_INPUT : st; r.end_bit = eb; r.end_hdr = eh; r.n_sym = ns; };
	for(;;) {
		const uint64_t hdr = b.pos();
		if(!resume) {
			r.safe_bit = hdr; r.safe_hdr = NONE; r.safe_sym = ns;
			if(hdr >= stop_bit) return finish(ST_STOP, hdr, NONE);
		}
		if(b.over()) return finish(E_INPUT, hdr, NONE);
		b.refill();
		const uint32_t fin = b.get(1), type = b.get(2);
		if(r.first_type < 0) r.first_type = (int)type;
		if(type == 3) return finish(E_BTYPE, hdr, NONE);
		if(type == 0) {
			b.drop(b.cnt & 7);
			const uint32_t len = b.get(16), nlen = b.get(16);
			if(b.over()) return finish(E_INPUT, hdr, NONE);
			if(len != (~nlen & 0xffffu)) return finish(E_STORED, hdr, NONE);
			const uint64_t q = b.pos() >> 3;
			if(q + len > n) return finish(E_INPUT, hdr, NONE);
			if(ns + len > cap) return finish(ST_FULL, hdr, NONE);
			for(uint32_t i = 0; i < len; i++) out[ns + i] = in[q + i];
			ns += len;
			b.init(in, n, (q + len) * 8);
			if(fin) return finish(ST_END, b.pos(), NONE);
			continue;
		}
		const int e = read_tables(b, (int)type, t, false);
		if(e) return finish(e, hdr, NONE);
		if(resume) { b.init(in, n, start_bit); resume = false; }
		for(;;) {
			if(b.over()) return finish(E_INPUT, hdr, NONE);
			if(ns + 258 > cap) {
				r.safe_bit = b.pos(); r.safe_hdr = hdr; r.safe_sym = ns;
				return finish(ST_FULL, b.pos(), hdr);
			}
			b.refill();
			int s = huff_decode(t.lit, b);
			if(s < 256) {
				if(s < 0) return finish(E_SYM, hdr, NONE);
				out[ns++] = (uint16_t)s;
				continue;
			}
			if(s == 256) break;
			s -= 257;
			if(s >= 29) return finish(E_SYM, hdr, NONE);
			// RFC 1951 3.2.5: length codes 257..284 and distance codes 4..29 come in groups of four and two per extra bit
			const int le = s < 8 || s == 28 ? 0 : (s >> 2) - 1;
			const uint32_t len = (s < 8 ? 3u + s : s == 28 ? 258u : ((4u + (s & 3)) << le) + 3u) + b.get(le);
			const int ds = huff_decode(t.dist, b);
			if(ds < 0 || ds >= 30) return finish(E_SYM, hdr, NONE);
			const int de = ds < 4 ? 0 : (ds >> 1) - 1;
			const uint32_t dist = (ds < 4 ? 1u + ds : ((2u + (ds & 1)) << de) + 1u) + b.get(de);
			if(dist <= ns) {
				// an overlapping copy repeats with period dist: read only symbols written before this match
				uint16_t* o = out + ns; const uint16_t* src = o - dist;
				if(dist >= len) for(uint32_t k = 0; k < len; k++) o[k] = src[k];
				else for(uint32_t k = 0, j = 0; k < len; k++) { o[k] = src[j]; if(++j == dist) j = 0; }
			} else {
				for(uint32_t k = 0; k < len; k++) {
					const int64_t from = (int64_t)ns + k - dist;
					out[ns + k] = from < 0 ? (uint16_t)(256 + WIN + from) : out[from];
				}
			}
			ns += len;
		}
		if(b.over()) return finish(E_INPUT, hdr, NONE);
		if(fin) return finish(ST_END, b.pos(), NONE);
	}
}

}  // namespace cfz
