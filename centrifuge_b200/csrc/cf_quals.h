// cf_quals.h -- FASTQ quality encodings (--phred33, --phred64, --solexa-quals, --int-quals), shared by the command line,
// the record-level reader (cf_host.cpp), the C ABI (cfb_ctx_set_quals) and the device tokeniser (k_tok_quals in
// cf_text.cuh).  One option state, one conversion per encoding, one Solexa -> Phred table.
//
// Reference behaviour restated (paths relative to the reference tree):
//   options, applied in command-line order   centrifuge.cpp:540-542,580-584,1038-1041: --phred64, --phred64-quals and
//                                            --solexa1.3-quals set phred64; --solexa-quals sets solexa; --int-quals and
//                                            --integer-quals set integer; --phred33 / --phred33-quals clear solexa and
//                                            phred64 (not integer)
//   character qualities                      charToPhred33 qual.h:105-146, applied to the kept characters only (those at
//                                            or after -5, pat.cpp:1042-1078); solexa wins over phred64; the character is
//                                            a signed char
//   integer qualities                        intToPhred33 qual.h:152-171 on atoi of every token, pat.cpp:997-1030
//   Solexa -> Phred                          solexaToPhred qual.h:45-49: 0 below -10, else a table (qual.cpp:57)
//
// The table is not copied: it is the published conversion round(10 log10(1 + 10^(Q/10))) for Q = -10 .. 255, which
// is Q itself from 10 up.  Below 10 it climbs by 0 or 1 per step, so the device holds it as one 20-bit mask of steps
// (solexa_steps) and counts them with a popcount.
//
// Where the reference is undefined this restatement clamps: a Solexa integer above 255 (past the end of the table)
// converts as 255, and a token whose value does not fit an int (atoi overflow) reads as INT_MAX or INT_MIN by its sign.
#ifndef CF_QUALS_H_
#define CF_QUALS_H_

#include <stdint.h>

#ifdef __CUDACC__
#define CFQ_HD __host__ __device__ __forceinline__
#else
#define CFQ_HD inline
#endif

#include <climits>
#include <cmath>
#include <string>

namespace cfb {

enum QualBits { QUAL_SOLEXA = 1, QUAL_PHRED64 = 2, QUAL_INTEGER = 4 };

struct Quals {
	bool solexa = false, phred64 = false, integer = false;
	bool is_default() const { return !solexa && !phred64 && !integer; }
	int bits() const { return (solexa ? QUAL_SOLEXA : 0) | (phred64 ? QUAL_PHRED64 : 0) | (integer ? QUAL_INTEGER : 0); }
	// one option name without its dashes: false when it is not a quality-encoding option
	bool apply(const std::string& o) {
		if(o == "phred64" || o == "phred64-quals" || o == "solexa1.3-quals") phred64 = true;
		else if(o == "solexa-quals") solexa = true;
		else if(o == "int-quals" || o == "integer-quals") integer = true;
		else if(o == "phred33" || o == "phred33-quals") { solexa = false; phred64 = false; }
		else return false;
		return true;
	}
};

// The published Solexa -> Phred conversion, in doubles (host only): 0 below -10
inline int solexa_formula(int q) {
	if(q < -10) return 0;
	return (int)std::floor(10.0 * std::log10(1.0 + std::pow(10.0, q / 10.0)) + 0.5);
}
// bit k (1 <= k < 20): solexa_formula(k - 10) exceeds solexa_formula(k - 11) by one; 0 when a step is not 0 or 1, or
// when the formula is not Q itself from 10 to 255 (tests/test_quals_host.py checks it is not)
inline uint32_t solexa_steps() {
	uint32_t m = 0;
	for(int k = 1; k < 20; k++) {
		const int d = solexa_formula(k - 10) - solexa_formula(k - 11);
		if(d != 0 && d != 1) return 0;
		m |= (uint32_t)d << k;
	}
	if(solexa_formula(-10) != 0) return 0;
	for(int q = 10; q <= 255; q++) if(solexa_formula(q) != q) return 0;
	return m;
}
// solexaToPhred: 0 below -10, the table from -10 to 9, Q itself from 10 up (255 past the table's end)
CFQ_HD int solexa_to_phred(int q, uint32_t steps) {
	if(q < -10) return 0;
	if(q >= 10) return q < 255 ? q : 255;
#ifdef __CUDA_ARCH__
	return __popc(steps & ((2u << (q + 10)) - 1u));
#else
	return __builtin_popcount(steps & ((2u << (q + 10)) - 1u));
#endif
}

// charToPhred33 of a kept quality byte under solexa / phred64 (not a space: the reader refuses those before).  The
// phred33 byte, or -1 where the reference refuses the character.
CFQ_HD int qual_from_char(uint32_t byte, bool solexa, bool phred64, uint32_t steps) {
	const int c = (int)(int8_t)(uint8_t)byte;
	if(solexa) return solexa_to_phred(c - 64, steps) + 33;      // never below 33: any byte is accepted
	if(phred64) return c < 64 ? -1 : c - 31;
	return c < 33 ? -1 : c;
}

// intToPhred33 of a token's atoi value: the phred33 value (it may pass 255 under solexa, where the reference keeps its
// low byte), or a value below 33 where the reference refuses it ("Saw negative Phred quality <v - 33>.")
CFQ_HD int qual_from_int(int v, bool solexa, uint32_t steps) {
	return solexa ? solexa_to_phred(v, steps) + 33 : (v <= 93 ? v : 93) + 33;
}

// atoi over [p, e) (one token: no ' ' inside): leading isspace, a sign, then digits up to the first non-digit,
// saturating at INT_MAX / INT_MIN
inline int qual_atoi(const char* p, const char* e) {
	while(p < e && (*p == ' ' || (*p >= 9 && *p <= 13))) p++;
	bool neg = false;
	if(p < e && (*p == '+' || *p == '-')) { neg = *p == '-'; p++; }
	long long v = 0;
	for(; p < e && *p >= '0' && *p <= '9'; p++) { v = v * 10 + (*p - '0'); if(v > (long long)INT_MAX + 1) v = (long long)INT_MAX + 1; }
	if(neg) return (int)(-v < INT_MIN ? INT_MIN : -v);
	return (int)(v > INT_MAX ? INT_MAX : v);
}

// error lines of the refusals, as the reference prints them (each ends the run with exit status 1)
inline std::string qual_char_error(uint32_t byte, bool phred64) {
	const int c = (int)(int8_t)(uint8_t)byte;
	if(phred64) return "Saw ASCII character " + std::to_string(c) + " but expected 64-based Phred qual.\nTry not specifying --solexa1.3-quals/--phred64-quals.";
	return "Saw ASCII character " + std::to_string(c) + " but expected 33-based Phred qual.";
}
inline std::string qual_int_error(int pq) { return "Saw negative Phred quality " + std::to_string(pq - 33) + "."; }

}  // namespace cfb

#endif  // CF_QUALS_H_
