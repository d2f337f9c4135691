// tests/native/longread_host.cpp -- TEST ONLY.  Compiles the long-unit logic of cf_logic.h (segmented chains and their join,
// post_search_long) for the host, next to the scalar search and post_search they must reproduce.
#include <cstring>
#include <string>
#include <vector>
#include "../../centrifuge_b200/csrc/cf_index.h"
#include "../../centrifuge_b200/csrc/cf_logic.h"

using namespace cfb;

struct LR { HostIndex h; IndexView v; };

extern "C" void* lr_load(const char* base) {
	LR* x = new LR();
	if(!load_cf_index(base, x->h).empty() || x->h.line_rate != 7) { delete x; return NULL; }
	const HostIndex& h = x->h; IndexView& v = x->v; memset(&v, 0, sizeof v);
	v.sides = (const uint64_t*)h.sides.data(); v.ftab = h.ftab.data(); v.eftab = h.eftab.data();
	v.len = h.len; v.zoff = h.zoff; v.zside = h.zoff / 384; v.zoffc = (uint32_t)(h.zoff % 384);
	for(int i = 0; i < 4; i++) v.fchr[i] = h.fchr[i];
	v.num_sides = h.num_sides; v.ftab_chars = h.ftab_chars;
	return x;
}
extern "C" void lr_free(void* p) { delete (LR*)p; }

static Params params(const LR* x, int khits, int min_hitlen) {
	Params p; p.khits = khits; p.min_hitlen = min_hitlen < 15 ? 15 : min_hitlen;
	p.ihits = (uint32_t)(khits > 5 ? khits : 5) * (x->h.compressed ? 4u : 40u);
	p.increment = (2 * p.min_hitlen <= 33) ? 10 : (2 * p.min_hitlen - 33);
	p.tree_traverse = 1; p.class_rank_slot = 0;
	return p;
}

struct Step {
	const IndexView& v; const uint8_t* fw; uint32_t len; int strand;
	void operator()(uint32_t cur, HitRec& h, uint32_t& nc, bool& done) { partial_search_scalar(v, fw, len, strand, cur, h, nc, done, nullptr); }
};

// The strand's hits by search_strand_scalar (a, *na) and by segmented chains of `seg` bases joined (b, *nb); both of capacity
// len + 2.  Returns the partial searches the join re-ran.
extern "C" unsigned long long lr_chains(void* hp, int min_hitlen, const uint8_t* fw, uint32_t len, int strand, uint32_t seg,
                                        HitRec* a, uint32_t* na, HitRec* b, uint32_t* nb) {
	const LR* x = (const LR*)hp; const Params p = params(x, 5, min_hitlen);
	*na = search_strand_scalar(x->v, p, fw, len, strand, a, len + 2, nullptr);
	const uint32_t nseg = (len + seg - 1) / seg;
	std::vector<HitRec> sh(len + 1); std::vector<uint32_t> sn(nseg + 1), sx(nseg + 1);
	Step step{x->v, fw, len, strand};
	for(uint32_t k = 0; k < nseg; k++) {
		const uint32_t start = k * seg, stop = start + seg < len ? start + seg : len;
		sn[k] = seg_chain(p, len, start, stop, step, sh.data() + start, &sx[k]);
	}
	unsigned long long re = 0;
	*nb = seg_join(p, len, seg, sh.data(), sn.data(), sx.data(), step, b, &re);
	return re;
}

// post_search (pruned = 0) or post_search_long (pruned = 1) on the lists of one mate, in place
extern "C" void lr_post(void* hp, int khits, int min_hitlen, const uint8_t* fw, uint32_t len, HitRec* F, uint32_t nF, HitRec* R, uint32_t nR, int pruned) {
	const LR* x = (const LR*)hp; const Params p = params(x, khits, min_hitlen);
	if(!pruned) { post_search(x->v, p, fw, len, F, nF, R, nR, nullptr); return; }
	std::vector<uint32_t> rcl(nR + 1);
	post_search_long(x->v, p, fw, len, F, nF, R, nR, rcl.data(), nullptr);
}

extern "C" int lr_is_chain(const HitRec* L, uint32_t n, uint32_t len) { return is_chain(L, n, len) ? 1 : 0; }
