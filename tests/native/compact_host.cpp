// tests/native/compact_host.cpp -- TEST ONLY.  Compiles the compact rank layout of cf_logic.h (cr_sb_entry, cr_convert_side,
// cr_lf, cr_bwt) for the host at several superblock spans, and the layout choice (choose_rank_layout).
#include <cstring>
#include <string>
#include <vector>
#include "../../centrifuge_b200/csrc/cf_index.h"
#include "../../centrifuge_b200/csrc/cf_logic.h"

using namespace cfb;

struct CH { HostIndex h; IndexView sides_view; };

extern "C" void* ch_load(const char* base) {
	CH* x = new CH();
	if(!load_cf_index(base, x->h).empty() || x->h.line_rate != 7) { delete x; return NULL; }
	const HostIndex& h = x->h; IndexView& v = x->sides_view; memset(&v, 0, sizeof v);
	v.sides = (const uint64_t*)h.sides.data();
	v.len = h.len; v.zoff = h.zoff; v.zside = h.zoff / 384; v.zoffc = (uint32_t)(h.zoff % 384);
	for(int i = 0; i < 4; i++) v.fchr[i] = h.fchr[i];
	v.num_sides = h.num_sides;
	return x;
}
extern "C" void ch_free(void* p) { delete (CH*)p; }
extern "C" uint64_t ch_rows(void* p) { return ((CH*)p)->h.len + 1; }

typedef uint64_t (*OracleLf)(const void*, uint64_t, int);
typedef int (*OracleBwt)(const void*, uint64_t);

// Converts a copy of the file's sides in place at superblock span 2^SB half-sides, as the loader does, then checks every row r in
// [0, len + 1] (the last is the exclusive bound of a full range) and every base c: the compact layout's LF(r, c) equals
// fchr[c] + the count of c in the oracle's BWT before r ('$' excluded), and for r <= len the oracle's LF and lf_scalar's over the
// file's sides; BWT[r] equals the oracle's.  Returns the number of mismatching rows; *first_bad receives the first.  The 64 bytes
// after the sides start as garbage, as on the device.
template <int SB> static uint64_t run(CH* x, OracleLf olf, OracleBwt obwt, const void* oh, uint64_t* first_bad) {
	const HostIndex& h = x->h;
	const uint64_t N = h.num_sides;
	std::vector<uint64_t> cr(N * 16 + 8, 0xdeadbeefdeadbeefull);
	memcpy(cr.data(), h.sides.data(), N * 128);
	std::vector<uint64_t> sb(cr_superblocks<SB>(N) * 4);
	for(uint64_t i = 0; i < sb.size() / 4; i++) cr_sb_entry<SB>(cr.data(), N, h.zoff, i, sb.data() + i * 4);
	for(uint64_t i = 0; i < N; i++) cr_convert_side<SB>(cr.data(), N, h.zoff, sb.data(), i);
	IndexView v = x->sides_view; v.sides = nullptr; v.cr = cr.data(); v.crsb = sb.data();
	const uint64_t n = h.len + 1;
	uint64_t bad = 0, cnt[4] = {0, 0, 0, 0};
	for(uint64_t r = 0; r <= n; r++) {
		bool ok = true;
		for(int c = 0; c < 4; c++) {
			const uint64_t got = cr_lf<SB>(v, r, c);
			ok &= got == h.fchr[c] + cnt[c];
			if(r < n) ok &= got == olf(oh, r, c) && got == lf_scalar(x->sides_view, r, c);
		}
		if(r < n) {
			const int b = obwt(oh, r);
			ok &= cr_bwt(v, r) == b;
			if(r != h.zoff) cnt[b]++;
		}
		if(!ok) { if(!bad) *first_bad = r; bad++; }
	}
	return bad;
}
extern "C" long long ch_check(void* p, int sb_shift, void* olf, void* obwt, void* oh, uint64_t* first_bad) {
	CH* x = (CH*)p; OracleLf f = (OracleLf)olf; OracleBwt g = (OracleBwt)obwt;
	switch(sb_shift) {
		case 1: return (long long)run<1>(x, f, g, oh, first_bad);
		case 2: return (long long)run<2>(x, f, g, oh, first_bad);
		case 3: return (long long)run<3>(x, f, g, oh, first_bad);
		case kCrSbShift: return (long long)run<kCrSbShift>(x, f, g, oh, first_bad);
	}
	return -1;
}
extern "C" uint64_t ch_num_sides(void* p) { return ((CH*)p)->h.num_sides; }
extern "C" uint64_t ch_zoff(void* p) { return ((CH*)p)->h.zoff; }

// IndexView's own path: lf_scalar / bwt_char with v.cr set (the default span), which the device's scalar LF runs
extern "C" void ch_view_lf(void* p, const uint64_t* rows, const uint8_t* chars, uint64_t n, uint64_t* out) {
	CH* x = (CH*)p; const HostIndex& h = x->h; const uint64_t N = h.num_sides;
	std::vector<uint64_t> cr(N * 16 + 8);
	memcpy(cr.data(), h.sides.data(), N * 128);
	std::vector<uint64_t> sb(cr_superblocks(N) * 4);
	for(uint64_t i = 0; i < sb.size() / 4; i++) cr_sb_entry(cr.data(), N, h.zoff, i, sb.data() + i * 4);
	for(uint64_t i = 0; i < N; i++) cr_convert_side(cr.data(), N, h.zoff, sb.data(), i);
	IndexView v = x->sides_view; v.sides = nullptr; v.cr = cr.data(); v.crsb = sb.data();
	for(uint64_t i = 0; i < n; i++) out[i] = lf_scalar(v, rows[i], chars[i] > 3 ? bwt_char(v, rows[i]) : chars[i]);
}

extern "C" int ch_choose(uint64_t free_b, uint64_t num_sides, uint64_t sample_b, uint64_t fixed_b, uint64_t headroom, int force_compact) {
	return choose_rank_layout(free_b, num_sides, sample_b, fixed_b, headroom, force_compact != 0);
}
extern "C" uint64_t ch_rank16_bytes(uint64_t num_sides) { return rank16_bytes_for(num_sides); }
extern "C" uint64_t ch_cr_bytes(uint64_t num_sides) { return cr_bytes_for(num_sides); }
