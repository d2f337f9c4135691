// Host build of centrifuge_b200/csrc/cf_quals.h for the quality-encoding tests: the conversions the record-level reader
// and k_tok_quals run, over many inputs at once.
#include "../../centrifuge_b200/csrc/cf_quals.h"

#include <cstring>

extern "C" uint32_t q_steps(void) { return cfb::solexa_steps(); }
extern "C" int q_solexa_formula(int q) { return cfb::solexa_formula(q); }

// every byte through qual_from_char under (solexa, phred64)
extern "C" void q_chars(int solexa, int phred64, int* out) {
	const uint32_t s = cfb::solexa_steps();
	for(int b = 0; b < 256; b++) out[b] = cfb::qual_from_char((uint32_t)b, solexa != 0, phred64 != 0, s);
}
// values lo .. hi through qual_from_int
extern "C" void q_ints(int solexa, int lo, int hi, int* out) {
	const uint32_t s = cfb::solexa_steps();
	for(int v = lo; v <= hi; v++) out[v - lo] = cfb::qual_from_int(v, solexa != 0, s);
}
extern "C" int q_atoi(const char* p) { return cfb::qual_atoi(p, p + strlen(p)); }
// 0 and the new state after applying `opt` to (solexa, phred64, integer) = bits, or -1 for a name it does not know
extern "C" int q_apply(int bits, const char* opt) {
	cfb::Quals q; q.solexa = bits & 1; q.phred64 = bits & 2; q.integer = bits & 4;
	if(!q.apply(opt)) return -1;
	return q.bits();
}
