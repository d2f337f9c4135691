// tests/native/walk8_rule.cpp -- TEST ONLY.  Checks walk8's range rule (cf_logic.h: walk8_steps, walk8_retry) against the
// host LF (lf_scalar on the file's sides) one base at a time, on random ranges and extensions of a real index.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include "../../centrifuge_b200/csrc/cf_index.h"
#include "../../centrifuge_b200/csrc/cf_logic.h"

using namespace cfb;

// k_build_walk8's entry of `row`, restated on the host: eight mapLF1 steps, stopping at the '$' row
static uint64_t entry(const IndexView& v, uint64_t row) {
	uint64_t r = row, chars = 0; uint32_t nv = 0;
	for(; nv < 8; nv++) {
		if(r == v.zoff) break;
		const int c = bwt_char(v, r);
		chars |= (uint64_t)c << (2 * nv);
		r = lf_scalar(v, r, c);
	}
	return (r & kWalkRowMask) | (chars << 40) | ((uint64_t)nv << 56);
}

// stats: 0 trials, 1 jumps accepted, 2 accepted from a range, 3 accepted from a range of width >= 5, 4 accepted where interior
// rows dropped out, 5 attempts rejected, 6 attempts that involved an end row within eight steps of '$', 7 retries checked
// before walk8_retry (all must fail), 8 mismatches (must be 0)
extern "C" long long w8_check(const char* base, uint64_t seed, uint32_t trials, unsigned long long* stats, char* err, size_t errlen) {
	HostIndex h;
	const std::string e = load_cf_index(base, h);
	if(!e.empty()) { strncpy(err, e.c_str(), errlen - 1); err[errlen - 1] = 0; return -1; }
	IndexView v; memset(&v, 0, sizeof v);
	v.sides = (const uint64_t*)h.sides.data(); v.len = h.len; v.zoff = h.zoff; v.zside = h.zoff / 384; v.zoffc = (uint32_t)(h.zoff % 384);
	for(int i = 0; i < 4; i++) v.fchr[i] = h.fchr[i];
	const uint64_t nrows = h.len + 1;
	if(nrows / 384 >= h.num_sides) { snprintf(err, errlen, "row %llu (a range's end) lies past the last side", (unsigned long long)nrows); return -1; }
	memset(stats, 0, 9 * sizeof *stats);
	std::mt19937_64 rng(seed);
	// rows whose walk meets '$' within eight steps: the rows of the eight text suffixes that start right after it
	std::vector<uint64_t> near;
	for(uint64_t r = 0; r < nrows; r++) if((entry(v, r) >> 56) < 8) near.push_back(r);
	if(near.size() != 8) { snprintf(err, errlen, "%zu rows reach '$' within eight steps, not 8", near.size()); return -1; }
	for(uint32_t t = 0; t < trials; t++) {
		stats[0]++;
		// a range: random, or with one end on a row near '$'; widths from 1 to a few hundred rows
		const uint32_t wsel = (uint32_t)(rng() % 4);
		uint64_t width = wsel == 0 ? 1 : wsel == 1 ? 2 + rng() % 3 : wsel == 2 ? 5 + rng() % 28 : 33 + rng() % 300;
		width = width < nrows ? width : nrows;
		uint64_t top = rng() % (nrows - width + 1);
		if(rng() % 8 == 0) { const uint64_t r = near[rng() % near.size()]; top = (rng() & 1) || r + 1 < width ? r : r + 1 - width; if(top + width > nrows) top = nrows - width; }
		uint64_t bot = top + width;
		// 16 read bases: the walk of one end row (or of a random row of the range), then point mutations and Ns
		int rd[16];
		{
			uint64_t r = (rng() & 1) ? top : (rng() & 1) ? bot - 1 : top + rng() % width;
			for(int j = 0; j < 16; j++) { const int c = r == v.zoff ? (int)(rng() % 4) : bwt_char(v, r); rd[j] = c; if(r != v.zoff) r = lf_scalar(v, r, c); }
			const uint32_t nmut = (uint32_t)(rng() % 3);
			for(uint32_t m = 0; m < nmut; m++) rd[rng() % 16] = (int)(rng() % 4);
			if(rng() % 10 == 0) rd[rng() % 16] = 4;
		}
		// one base at a time: range[j] after j bases (empty once it dies; an N ends the walk)
		uint64_t T[17], B[17]; T[0] = top; B[0] = bot; int alive = 0;
		for(int j = 0; j < 16; j++) {
			const int c = rd[j];
			if(c > 3) break;
			const uint64_t nt = lf_scalar(v, T[j], c), nb = lf_scalar(v, B[j], c);
			if(nb <= nt) break;
			T[j + 1] = nt; B[j + 1] = nb; alive = j + 1;
		}
		// a jump attempted after j bases, j = 0..8, on whatever range the walk holds then
		uint32_t retry = 0;
		for(int j = 0; j <= 8 && j <= alive; j++) {
			uint64_t win = 0; uint32_t nwin = 0;
			for(int k = 0; k < 8; k++) { if(rd[j + k] > 3) nwin |= 1u << k; else win |= (uint64_t)rd[j + k] << (2 * k); }
			const uint64_t et = entry(v, T[j]), eb = entry(v, B[j] - 1);
			const uint32_t st = walk8_steps(et, win, nwin), sb = walk8_steps(eb, win, nwin);
			if((et >> 56) < 8 || (eb >> 56) < 8) stats[6]++;
			if((uint32_t)j < retry) {      // walk8_retry of the attempt at 0 says this one fails
				stats[7]++;
				if((st & sb) == 8u) stats[8]++;
			}
			if((st & sb) == 8u) {
				stats[1]++;
				const uint64_t nt = et & kWalkRowMask, nb = (eb & kWalkRowMask) + 1;
				if(alive < j + 8 || T[j + 8] != nt || B[j + 8] != nb) stats[8]++;
				if(B[j] - T[j] > 1) stats[2]++;
				if(B[j] - T[j] >= 5) stats[3]++;
				if(alive >= j + 8 && B[j + 8] - T[j + 8] < B[j] - T[j]) stats[4]++;
			} else {
				stats[5]++;
				if(j == 0) retry = walk8_retry(st, sb);
			}
		}
	}
	return (long long)stats[8];
}
