// tests/native/fastpath_host.cpp -- TEST ONLY.  The rank16 search path's information loss, on the host: the exact hit lists of
// the scalar search (search_strand_scalar) are degraded the way k_search_t stores them -- hits the death bitmap can end lose
// their SA range (kUnk), and with min_hitlen >= kLongLen the short hits are not stored -- and then go through the rules by which
// load_unit and k_prep restore what matters (list_dropped, list_needs_regen, list_needs_exact_ranges in cf_logic.h, the code
// the kernels run) and the rest of the per-unit logic.  The records must be the exact search's, which are the oracle's.
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <set>
#include "../../centrifuge_b200/csrc/cf_index.h"
#include "../../centrifuge_b200/csrc/cf_logic.h"

using namespace cfb;

struct FP { HostIndex h; IndexView v; std::vector<uint8_t> excl; std::vector<uint64_t> host; int K; int degrade; };

static void expand(const HostIndex& h, const uint64_t* ids, uint64_t n, std::set<uint64_t>& out) {
	if(!n) return;
	for(size_t i = 0; i < h.nodes.size(); i++) {
		uint64_t t = h.nodes[i].taxid;
		for(;;) {
			bool f = false; for(uint64_t k = 0; k < n; k++) if(ids[k] == t) f = true;
			if(f) { out.insert(h.nodes[i].taxid); break; }
			const TaxNode* nd = h.find_node(t);
			if(!nd || nd->parent == t) break;
			t = nd->parent;
		}
	}
}

extern "C" void* fp_load(const char* base, char* err, size_t errlen) {
	FP* x = new FP();
	std::string e = load_cf_index(base, x->h);
	if(e.empty() && x->h.line_rate != 7) e = "lineRate 7 only";
	if(!e.empty()) { strncpy(err, e.c_str(), errlen - 1); err[errlen - 1] = 0; delete x; return NULL; }
	const HostIndex& h = x->h; IndexView& v = x->v; memset(&v, 0, sizeof v);
	v.sides = (const uint64_t*)h.sides.data(); v.ftab = h.ftab.data(); v.eftab = h.eftab.data();
	v.sample16 = h.wide_sample ? NULL : h.sample16.data(); v.sample32 = h.wide_sample ? h.sample32.data() : NULL;
	v.brow = h.brow.data(); v.bseq = h.bseq.data(); v.bbits = h.bbits.data();
	v.seq_taxid = h.seq_taxid.data(); v.seq_path = h.seq_path.data(); v.paths = h.paths.data();
	v.len = h.len; v.zoff = h.zoff; v.zside = h.zoff / 384; v.zoffc = (uint32_t)(h.zoff % 384);
	for(int i = 0; i < 4; i++) v.fchr[i] = h.fchr[i];
	v.last_boundary = h.last_boundary; v.num_sides = h.num_sides; v.n_boundaries = (uint32_t)h.brow.size();
	v.n_seqs = (uint32_t)h.seq_taxid.size(); v.off_rate = h.off_rate; v.ftab_chars = h.ftab_chars; v.bshift = h.bshift;
	// the K-mer table's K as the loader picks it with HBM to spare (the death bitmap's hits end at K .. K + 2 bases)
	int K = h.ftab_chars;
	while(K < 15 && (4ull << (2 * K)) <= h.len / 4) K++;
	x->K = K; x->degrade = 1;
	return x;
}
extern "C" void fp_free(void* p) { delete (FP*)p; }
extern "C" int fp_kmer_chars(void* p) { return ((FP*)p)->K; }
extern "C" void fp_set_degrade(void* p, int degrade) { ((FP*)p)->degrade = degrade; }

struct OParams { int khits, min_hitlen, tree_traverse, class_rank_slot; const uint64_t* host; size_t n_host; const uint64_t* excl; size_t n_excl; };

// Whether the death bitmap can end the partial search of hit h: the K-mer gather is taken with the bitmap only when
// min_hitlen >= K + 3 and K + 3 bases without an N are left, and then it ends searches whose range dies after K .. K + 2 bases.
static bool bitmap_can_end(const Params& p, int K, const uint8_t* fw, uint32_t len, int strand, const HitRec& h) {
	const uint32_t fd = (uint32_t)K + 3;
	if(p.min_hitlen < fd || h.top == kOff || h.len < (uint32_t)K || h.len > (uint32_t)K + 2 || (uint64_t)h.bwoff + fd > len) return false;
	for(uint32_t d = h.bwoff; d < h.bwoff + fd; d++) if(seq_at(fw, len, strand, len - 1 - d) > 3) return false;
	return true;
}

// The oracle's cfo_classify signature.  fp_set_degrade 0: the exact lists (hostlogic.cpp's classification); 1 (the default):
// the rank16 path's lists and rules.  stats (16 words): [0] hits blanked to kUnk, [1] short hits not stored, [2] lists load_unit emptied,
// [3] lists regenerated, [4] lists given exact ranges, [5] kUnk hits still in a list when it is sorted, [6] counted hits
// carrying kRowSameTs.
extern "C" long long fp_classify(void* hp, const OParams* op, const uint8_t* bases, const uint64_t* off1, const uint32_t* len1,
                                 const uint64_t* off2, const uint32_t* len2, const uint8_t* flags, size_t n,
                                 uint32_t* out_n, OutRec* out, size_t cap, unsigned long long* stats) {
	FP* x = (FP*)hp; const HostIndex& h = x->h; const int degrade = x->degrade;
	Params p; p.khits = op->khits; p.min_hitlen = op->min_hitlen < 15 ? 15 : op->min_hitlen;
	p.ihits = (uint32_t)std::max(op->khits, 5) * (h.compressed ? 4u : 40u);
	p.increment = (2 * p.min_hitlen <= 33) ? 10 : (2 * p.min_hitlen - 33);
	p.tree_traverse = op->tree_traverse; p.class_rank_slot = (uint32_t)op->class_rank_slot & 0xff;
	std::set<uint64_t> hs, es; expand(h, op->host, op->n_host, hs); expand(h, op->excl, op->n_excl, es);
	IndexView v = x->v;
	x->excl.assign(h.seq_taxid.size(), 0);
	if(!es.empty()) { for(size_t i = 0; i < x->excl.size(); i++) x->excl[i] = es.count(h.seq_taxid[i]) ? 1 : 0; v.seq_excluded = x->excl.data(); }
	x->host.assign(hs.begin(), hs.end());
	if(!x->host.empty()) { v.host_taxids = x->host.data(); v.n_host = (uint32_t)x->host.size(); }
	const bool keep_short = p.min_hitlen < kLongLen;      // k_search_t stores every hit below kLongLen
	size_t total = 0;
	for(size_t i = 0; i < n; i++) {
		uint8_t fl = flags ? flags[i] : 1;
		const bool pair = off2 && len2 && (fl & 4);
		if(!pair) fl &= 1;
		UnitHits u; u.n_mates = 0; const uint8_t* fw[2];
		std::vector<HitRec> exact[2][2], store[2][2];
		for(int m = 0; m < (pair ? 2 : 1); m++) {
			if(!((fl >> m) & 1)) continue;
			const uint32_t len = m == 0 ? len1[i] : len2[i];
			if(len == 0) continue;
			const int r = u.n_mates++;
			fw[r] = bases + (m == 0 ? off1[i] : off2[i]); u.rdlen[r] = len;
			uint32_t raw[2], found[2];
			for(int s = 0; s < 2; s++) {
				exact[r][s].resize(len + 2);
				found[s] = search_strand_scalar(v, p, fw[r], len, s, exact[r][s].data(), len + 2, nullptr);
				exact[r][s].resize(found[s]);
				store[r][s].clear();
				bool nolong = true;
				for(HitRec hr : exact[r][s]) {
					if(hr.len >= p.min_hitlen) nolong = false;
					if(!degrade) { store[r][s].push_back(hr); continue; }
					if(bitmap_can_end(p, x->K, fw[r], len, s, hr)) { hr.top = hr.bot = kUnk; stats[0]++; }
					if(keep_short || hr.len >= kLongLen) store[r][s].push_back(hr);
					else stats[1]++;
				}
				raw[s] = nh_pack((uint32_t)store[r][s].size(), found[s], nolong);
				u.L[r][s] = store[r][s].data(); u.n[r][s] = (uint32_t)store[r][s].size();
			}
			if(!degrade) continue;
			for(int s = 0; s < 2; s++) if(list_dropped(raw, s)) { if(u.n[r][s]) stats[2]++; u.n[r][s] = 0; }
			if(!keep_short) for(int s = 0; s < 2; s++) {
				if(!list_needs_regen(u.n[r][s], u.n[r][s ^ 1], found[s])) continue;
				store[r][s] = exact[r][s]; u.L[r][s] = store[r][s].data(); u.n[r][s] = found[s]; stats[3]++;
			}
			for(int s = 0; s < 2; s++) {
				if(!list_needs_exact_ranges(p, u.L[r][s], u.n[r][s], u.n[r][s ^ 1])) continue;
				stats[4]++;
				for(uint32_t k = 0; k < u.n[r][s]; k++) {
					HitRec& hr = u.L[r][s][k];
					if(hr.top != kUnk) continue;
					HitRec t; uint32_t nc; bool dn;
					partial_search_scalar(v, fw[r], len, s, hr.bwoff, t, nc, dn, nullptr);
					hr.top = t.top; hr.bot = t.bot;
				}
			}
			for(int s = 0; s < 2; s++) for(uint32_t k = 0; k < u.n[r][s]; k++) stats[5] += u.L[r][s][k].top == kUnk;
		}
		uint32_t no = 0;
		std::vector<OutRec> recs;
		if(u.n_mates > 0) {
			for(int r = 0; r < u.n_mates; r++) post_search(v, p, fw[r], u.rdlen[r], u.L[r][0], u.n[r][0], u.L[r][1], u.n[r][1], nullptr);
			SortAndCount sc(p, u); for_each_visit(p, u, sc);
			std::vector<uint64_t> rows(sc.rows + 1); std::vector<uint32_t> ids(sc.rows + 1);
			EmitRows er(p, u, rows.data()); for_each_visit(p, u, er);
			if(er.k != sc.rows) return -2;
			for(uint64_t k = 0; k < sc.rows; k++) { ids[k] = resolve_scalar(v, rows[k] & kRowMask, nullptr); stats[6] += (rows[k] & kRowSameTs) != 0; }
			std::vector<Entry> ent(sc.rows + 1); std::vector<TaxCnt> tc(sc.rows + 1); recs.resize(sc.rows + 1);
			const uint32_t nmap = score_plan(v, p, rows.data(), ids.data(), sc.rows, ent.data());
			no = reduce_and_emit(v, p, u.n_mates == 2, ent.data(), nmap, tc.data(), recs.data());
		}
		out_n[i] = no;
		if(total + no > cap) return -1;
		for(uint32_t k = 0; k < no; k++) out[total++] = recs[k];
	}
	return (long long)total;
}

// The time-stamp case by hand: a pair, -k 1.  Mate 1's one visited list holds a counted 30-base hit of one row, so it ends
// through its `break` (maxG = 1).  Mate 2's visited list holds, in chain order, an uncounted 12-base hit whose range holds three
// rows (size / len = 3/12) and a counted 18-base hit of one row (1/18): sorted, the counted hit comes first and shares mate 1's
// time stamp (kRowSameTs).  blank = 1 stores the 12-base hit as the death bitmap leaves it (kUnk, size 0), which sorts it first;
// restore = 1 then applies list_needs_exact_ranges and gives the lists that need it their true ranges back.  Writes the rows
// EmitRows plans (at most cap), needs[mate] = list_needs_exact_ranges of the visited lists, and returns the number of rows.
extern "C" int fp_ts_case(int min_hitlen, int blank, int restore, uint64_t* rows, uint32_t cap, int* needs) {
	Params p; p.khits = 1; p.min_hitlen = (uint32_t)min_hitlen; p.ihits = 200; p.increment = 10; p.tree_traverse = 1; p.class_rank_slot = 0;
	HitRec a[1] = {{1000, 1001, 0, 30}};
	const HitRec short_true = {5000, 5003, 0, 12};
	HitRec b[2] = {short_true, {7000, 7001, 13, 18}};
	if(blank) b[0].top = b[0].bot = kUnk;
	UnitHits u; u.n_mates = 2; u.rdlen[0] = u.rdlen[1] = 40;
	u.L[0][0] = a; u.n[0][0] = 1; u.L[0][1] = nullptr; u.n[0][1] = 0;
	u.L[1][0] = b; u.n[1][0] = 2; u.L[1][1] = nullptr; u.n[1][1] = 0;
	needs[0] = list_needs_exact_ranges(p, a, 1, 0); needs[1] = list_needs_exact_ranges(p, b, 2, 0);
	if(restore && needs[1] && b[0].top == kUnk) { b[0].top = short_true.top; b[0].bot = short_true.bot; }
	SortAndCount sc(p, u); for_each_visit(p, u, sc);
	if(sc.rows > cap) return -1;
	EmitRows er(p, u, rows); for_each_visit(p, u, er);
	return (int)er.k;
}
