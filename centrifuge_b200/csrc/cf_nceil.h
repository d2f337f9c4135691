// cf_nceil.h -- the per-read N ceiling (--n-ceil), shared by the command line, the record-level reader (cf_host.cpp),
// the C ABI (cfb_ctx_set_n_ceil) and the device tokeniser (k_tok_bases in cf_text.cuh).  One parser, one evaluation.
//
// Reference behaviour restated (paths relative to the reference tree):
//   --n-ceil tokens -> "NCEIL=" policy     centrifuge.cpp:1323-1347 (1 token -> C,<x>; > 3 or 0 tokens are errors)
//   NCEIL= -> SimpleFunc                   aligner_seed_policy.cpp:47-75,525-530 (PARSE_FUNC), simple_func.cpp:25-41
//   default L,0,0.15, min 0, max DBL_MAX   aligner_seed_policy.cpp:296-298 (SimpleFunc::init(type, I, X, C, L))
//   f<size_t>(len)                         simple_func.h:85-108: max(I, min(X, C + L * g(len))), DBL_MAX -> SIZE_MAX
//   the read passes iff #Ns <= ceiling     Scoring::nFilter scoring.cpp:104-117; mates apart (ncatpair is false,
//                                          DEFAULT_N_CAT_PAIR scoring.h:67, and no option sets it)
//
// --n-ceil takes at most three tokens, so the minimum stays 0 and the maximum DBL_MAX: the ceiling is never negative,
// and (size_t) of a double is only ever taken of a value in [0, DBL_MAX).  For values of 2^64 and up that conversion
// is what gcc emits for x86-64 without AVX-512 (cvttsd2si of x - 2^63, then bit 63 flipped), which yields 0; the
// reference binary is built that way, so nceil_to_size() restates it.
//
// Arithmetic: one multiply and one add, never contracted into an FMA (the _rn intrinsics on the device,
// -ffp-contract=off on the host), so that the device gives the host's double for every length.  sqrt is correctly
// rounded on both sides.  The device's double log differs from glibc's in the last bit at about one length in 18 000
// below 2^31 (never by more; tests/test_gpu_n_ceil.py counts them), so the device evaluates the log ceiling at the
// neighbouring doubles too and hands the read to the host where they disagree.
//
// Without --n-ceil the product keeps its historical coefficient, the double 0.15 (`--n-ceil L,0,0.15` parses to exactly
// that).  The reference's built-in default is the float 0.15f widened to a double; the two give the same ceiling for
// every length below 8 388 613 bases.  A parsed --n-ceil starts from the reference's 0.15f (nceil_policy_init).
#ifndef CF_NCEIL_H_
#define CF_NCEIL_H_

#include <stdint.h>

#ifdef __CUDACC__
#define CFN_HD __host__ __device__ __forceinline__
#else
#define CFN_HD inline
#endif

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <sstream>
#include <string>
#include <vector>

namespace cfb {

enum NCeilType { NCEIL_CONST = 1, NCEIL_LINEAR = 2, NCEIL_SQRT = 3, NCEIL_LOG = 4 };   // SIMPLE_FUNC_* simple_func.h:29-32

struct NCeil {
	int type = NCEIL_LINEAR;
	double c = 0.0, l = 0.15, mn = 0.0, mx = DBL_MAX;
	bool is_default() const { return type == NCEIL_LINEAR && c == 0.0 && l == 0.15 && mn == 0.0 && mx == DBL_MAX; }
};

// What the reference's policy parser starts the first --n-ceil from: SimpleFunc::init(L, 0, DBL_MAX, 0, 0.15f)
// (aligner_seed_policy.cpp:296-298, DEFAULT_N_CEIL_LINEAR scoring.h:63).  The coefficient is the float 0.15f widened,
// 0.15000000596..., so every value that leaves it unset (`L,<c>`, `S,<c>`, `G,<c>`, `L,abc`) takes that one.
inline NCeil nceil_policy_init() { NCeil f; f.l = (double)0.15f; return f; }

// (size_t)x as the x86-64 reference binary computes it for x in [0, DBL_MAX)
CFN_HD uint64_t nceil_to_size(double x) {
	const double two63 = 9223372036854775808.0;
	if(!(x >= two63)) return (uint64_t)(int64_t)x;
	const double y = x - two63;           // exact for x < 2^64
	if(y >= two63) return 0;              // cvttsd2si gives 0x8000000000000000, the flip of bit 63 clears it
	return (uint64_t)(int64_t)y ^ 0x8000000000000000ull;
}

// max(I, min(X, C + L * g)) as size_t, for g = the function of the length; `r` gets the clamped double
CFN_HD uint64_t nceil_of(double g, double c, double l, double mn, double mx, double* r_out = nullptr) {
#ifdef __CUDA_ARCH__
	const double v = __dadd_rn(c, __dmul_rn(l, g));
#else
	const double v = c + l * g;
#endif
	const double lo = v < mx ? v : mx;          // std::min(X, v): v when v < X, else X (a NaN gives X)
	const double r = mn < lo ? lo : mn;         // std::max(I, lo)
	if(r_out) *r_out = r;
	if(r == DBL_MAX) return UINT64_MAX;
	if(r == DBL_MIN) return 0;
	return nceil_to_size(r);
}

// SimpleFunc::f<size_t>((double)len).  On the device the log ceiling is exact only where the device's log, off from
// glibc's by at most one unit in the last place, cannot move it: `sure` is cleared for a length where the ceilings of
// the log's two neighbouring doubles differ (the caller then hands the read to the host).
CFN_HD uint64_t nceil_eval(int type, double c, double l, double mn, double mx, uint64_t len, bool* sure = nullptr) {
	const double x = (double)len;
	if(sure) *sure = true;
	double g;
#ifdef __CUDA_ARCH__
	if(type == NCEIL_CONST) g = 0.0;
	else if(type == NCEIL_LINEAR) g = x;
	else if(type == NCEIL_SQRT) g = __dsqrt_rn(x);
	else {
		g = log(x);
		double r0, r1;
		const uint64_t k0 = nceil_of(nextafter(g, -INFINITY), c, l, mn, mx, &r0), k1 = nceil_of(nextafter(g, INFINITY), c, l, mn, mx, &r1);
		if(sure && (k0 != k1 || (r0 < 18446744073709551616.0) != (r1 < 18446744073709551616.0))) *sure = false;
	}
#else
	if(type == NCEIL_CONST) g = 0.0;
	else if(type == NCEIL_LINEAR) g = x;
	else if(type == NCEIL_SQRT) g = std::sqrt(x);
	else g = std::log(x);
#endif
	return nceil_of(g, c, l, mn, mx);
}

// the N filter's verdict on a mate of `len` bases with `ns` Ns; `sure` as in nceil_eval
CFN_HD bool nceil_pass(int type, double c, double l, double mn, double mx, uint64_t len, uint64_t ns, bool* sure = nullptr) {
	return ns <= nceil_eval(type, c, l, mn, mx, len, sure);
}

inline uint64_t nceil_eval(const NCeil& f, uint64_t len) { return nceil_eval(f.type, f.c, f.l, f.mn, f.mx, len); }

// nFilter + lenfilt of one mate of codes 0..4 (centrifuge.cpp:2559-2584)
inline bool nceil_filter(const NCeil& f, const uint8_t* s, size_t n) {
	if(n < 2) return false;
	const uint64_t maxns = nceil_eval(f, n);
	uint64_t ns = 0;
	for(size_t i = 0; i < n; i++) if(s[i] == 4 && ++ns > maxns) return false;
	return true;
}

// Hit-list capacity of a strand of a mate of up to `maxlen` bases under the ceiling f: a partial search that meets an N
// within its next bases ends in a null hit (hi_aligner.h:903-1031), so a list holds up to about one entry per N that
// may pass plus one per 10 bases.  The ceiling is monotone in the length, so its largest value over the lengths that
// pass (>= 2) is at an end.  Never below the default's maxlen / 4 + 8, never above one entry per base (+ 2).
inline uint32_t nceil_full_cap(const NCeil& f, uint32_t maxlen) {
	const uint64_t base = maxlen / 4 + 8, top = (uint64_t)maxlen + 2;
	uint64_t ns = std::max(nceil_eval(f, 2), nceil_eval(f, maxlen));
	ns = std::min<uint64_t>(ns, maxlen);
	return (uint32_t)std::min(top, std::max(base, ns + maxlen / 10 + 8));
}

// --n-ceil <func> applied on top of f (nceil_policy_init() for the first one): false with the reference's first error line in `err` (its exit code is 1).  `setting` is the place of
// this NCEIL= in the reference's policy string: SEED, DPS, ROUNDS and IVAL come first, so the first --n-ceil is the 5th.
inline bool nceil_parse(const std::string& arg, NCeil& f, std::string& err, int setting = 5) {
	// tokenize(arg, ",", args) tokenize.h:34-51: the first token is kept even when empty (so "" is one empty token),
	// later runs of commas count as one, and a trailing comma adds nothing
	std::vector<std::string> args;
	{
		size_t last = 0, pos = arg.find_first_of(',', last);
		while(pos != std::string::npos || last != std::string::npos) {
			args.push_back(arg.substr(last, pos == std::string::npos ? std::string::npos : pos - last));
			last = arg.find_first_not_of(',', pos);
			pos = arg.find_first_of(',', last);
		}
	}
	if(args.size() > 3) {
		std::ostringstream os; os << "Error: expected 3 or fewer comma-separated arguments to --n-ceil option, got " << args.size();
		err = os.str(); return false;
	}
	if(args.empty()) { err = "Error: expected at least one argument to --n-ceil option"; return false; }
	std::string s = args.size() == 1 ? "C," + args[0] : (args.size() == 2 ? args[0] + "," + args[1] : args[0] + "," + args[1] + "," + args[2]);
	// PARSE_FUNC: getline-split on ',', then the type and `istringstream >> double` for each coefficient (0 on failure)
	std::vector<std::string> ctoks; { std::istringstream css(s); std::string t; while(std::getline(css, t, ',')) ctoks.push_back(t); }
	for(size_t i = 0; i < ctoks.size(); i++) if(ctoks[i].empty()) {      // aligner_seed_policy.cpp:355-361
		std::ostringstream os; os << "Error parsing alignment policy setting " << setting << "; token " << i + 1 << " on RHS had length=0";
		err = os.str(); return false;
	}
	NCeil r = f;
	if(ctoks.size() >= 1) {
		const std::string& t = ctoks[0];
		if(t == "C" || t == "Constant") r.type = NCEIL_CONST;
		else if(t == "L" || t == "Linear") r.type = NCEIL_LINEAR;
		else if(t == "S" || t == "Sqrt") r.type = NCEIL_SQRT;
		else if(t == "G" || t == "Log") r.type = NCEIL_LOG;
		else { err = "Error: Bad function type '" + t + "'.  Should be C (constant), L (linear), S (square root) or G (natural log)."; return false; }
	}
	double* dst[4] = {&r.c, &r.l, &r.mn, &r.mx};
	for(size_t k = 1; k < ctoks.size() && k <= 4; k++) { double v; std::istringstream ss(ctoks[k]); ss >> v; *dst[k - 1] = v; }
	f = r;
	return true;
}

}  // namespace cfb

#endif  // CF_NCEIL_H_
