// Host build of centrifuge_b200/csrc/cf_nceil.h for the --n-ceil tests: the ceiling the device tokeniser evaluates,
// compiled with -ffp-contract=off as the library is, over many lengths at once, and the shared parser.
#include "../../centrifuge_b200/csrc/cf_nceil.h"

#include <cstring>

extern "C" void nc_eval_many(int type, double c, double l, const uint64_t* len, uint64_t n, uint64_t* out) {
	for(uint64_t i = 0; i < n; i++) out[i] = cfb::nceil_eval(type, c, l, 0.0, DBL_MAX, len[i]);
}

extern "C" uint32_t nc_full_cap(int type, double c, double l, uint32_t maxlen) {
	cfb::NCeil f; f.type = type; f.c = c; f.l = l;
	return cfb::nceil_full_cap(f, maxlen);
}

// 0 and the function, or 1 and the error line
extern "C" int nc_parse(const char* spec, int* type, double* c, double* l, char* err, int err_cap) {
	cfb::NCeil f = cfb::nceil_policy_init(); std::string e;
	if(!cfb::nceil_parse(spec, f, e)) { strncpy(err, e.c_str(), err_cap - 1); err[err_cap - 1] = 0; return 1; }
	*type = f.type; *c = f.c; *l = f.l;
	return 0;
}
