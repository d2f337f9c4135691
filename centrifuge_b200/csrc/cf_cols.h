// cf_cols.h -- the columns of the classification TSV (--tab-fmt-cols), shared by the command line, the C ABI, the
// host formatter (cf_host.cpp) and the device formatter (cf_text.cuh).  One table of names, one parser, one row
// composer: every consumer formats a row by handing emit_row() its values and a byte sink.
//
// Reference behaviour restated (paths relative to the reference tree):
//   names -> fields                     centrifuge.cpp:483-518 (col_name_map), FIELD_DEF aln_sink.h:2253-2273
//   list parsing + error                centrifuge.cpp:268-281 (tokenize on ",", tokenize.h:34-51)
//   header line                         centrifuge.cpp:2985-2992
//   field text                          AlnSinkSam::appendMate aln_sink.h:2280-2337
#ifndef CF_COLS_H_
#define CF_COLS_H_

#include <stdint.h>

#ifdef __CUDACC__
#define CFC_HD __host__ __device__ __forceinline__
#else
#define CFC_HD inline
#endif

#include <string>
#include <vector>

namespace cfb {

// FIELD_DEF values (aln_sink.h:2253-2273)
enum ColField : uint8_t {
	COL_PLACEHOLDER = 0, COL_PLACEHOLDER_STAR, COL_PLACEHOLDER_ZERO, COL_READ_ID, COL_SEQ_ID, COL_TAX_ID, COL_TAX_RANK,
	COL_TAX_NAME, COL_SCORE, COL_SCORE2, COL_HIT_LENGTH, COL_QUERY_LENGTH, COL_NUM_MATCHES, COL_SEQ, COL_SEQ1, COL_SEQ2,
	COL_QUAL, COL_QUAL1, COL_QUAL2, COL_N_FIELDS
};
static const int kTextMaxCols = 64;       // longest list the device formatter takes; longer lists are formatted on the host
static const char* const kDefaultCols = "readID,seqID,taxID,score,2ndBestScore,hitLength,queryLength,numMatches";

struct ColName { const char* name; uint8_t field; };
static const ColName kColNames[] = {
	{"readID", COL_READ_ID}, {"seqID", COL_SEQ_ID}, {"taxLevel", COL_TAX_RANK}, {"taxRank", COL_TAX_RANK}, {"taxID", COL_TAX_ID},
	{"taxName", COL_TAX_NAME}, {"score", COL_SCORE}, {"2ndBestScore", COL_SCORE2}, {"hitLength", COL_HIT_LENGTH},
	{"queryLength", COL_QUERY_LENGTH}, {"numMatches", COL_NUM_MATCHES}, {"readSeq", COL_SEQ}, {"readQual", COL_QUAL},
	// SAM names
	{"QNAME", COL_READ_ID}, {"FLAG", COL_PLACEHOLDER_ZERO}, {"RNAME", COL_TAX_ID}, {"POS", COL_PLACEHOLDER_ZERO},
	{"MAPQ", COL_PLACEHOLDER_ZERO}, {"CIGAR", COL_PLACEHOLDER}, {"RNEXT", COL_SEQ_ID}, {"PNEXT", COL_PLACEHOLDER_ZERO},
	{"TLEN", COL_QUERY_LENGTH}, {"SEQ", COL_SEQ}, {"QUAL", COL_QUAL},
	// one mate each
	{"SEQ1", COL_SEQ1}, {"SEQ2", COL_SEQ2}, {"QUAL1", COL_QUAL1}, {"QUAL2", COL_QUAL2},
	{"readSeq1", COL_SEQ1}, {"readSeq2", COL_SEQ2}, {"readQual1", COL_QUAL1}, {"readQual2", COL_QUAL2},
};

CFC_HD uint32_t col_mask(const uint8_t* cols, uint32_t n) { uint32_t m = 0; for(uint32_t i = 0; i < n; i++) m |= 1u << cols[i]; return m; }
static const uint32_t kColSeqBits = (1u << COL_SEQ) | (1u << COL_SEQ1) | (1u << COL_SEQ2);
static const uint32_t kColQualBits = (1u << COL_QUAL) | (1u << COL_QUAL1) | (1u << COL_QUAL2);

// A parsed --tab-fmt-cols list (host code): the names as given (they are the header) and their fields.
struct ColList {
	std::vector<std::string> names; std::vector<uint8_t> fields;
	// parse_col_fmt: tokens between commas, a run of commas counts as one separator, a trailing one ends the list, a
	// leading one (or an empty list) gives an empty name.  Returns false with the reference's message for an unknown name.
	bool parse(const std::string& arg, std::string& err) {
		std::vector<std::string> tok;
		size_t last = 0, pos = arg.find_first_of(',', last);
		while(pos != std::string::npos || last != std::string::npos) {
			tok.push_back(arg.substr(last, pos == std::string::npos ? std::string::npos : pos - last));
			last = arg.find_first_not_of(',', pos);
			pos = arg.find_first_of(',', last);
		}
		std::vector<uint8_t> f;
		for(size_t i = 0; i < tok.size(); i++) {
			int code = -1;
			for(size_t k = 0; k < sizeof(kColNames) / sizeof(kColNames[0]); k++) if(tok[i] == kColNames[k].name) { code = kColNames[k].field; break; }
			if(code < 0) { err = "Column definition " + tok[i] + " invalid."; return false; }
			f.push_back((uint8_t)code);
		}
		names.swap(tok); fields.swap(f);
		return true;
	}
	std::string header() const { std::string h; for(size_t i = 0; i < names.size(); i++) { if(i) h += '\t'; h += names[i]; } return h + "\n"; }
	std::string spec() const { std::string h; for(size_t i = 0; i < names.size(); i++) { if(i) h += ','; h += names[i]; } return h; }   // parses back to this list
	int index_of(uint8_t field) const { for(size_t i = 0; i < fields.size(); i++) if(fields[i] == field) return (int)i; return -1; }
	uint32_t mask() const { return col_mask(fields.data(), (uint32_t)fields.size()); }
};

// Everything a row can print.  Strings are not terminated; base codes are 0..4; qual[m] == NULL means a FASTA read,
// whose qualities are qn[m] times 'I' (pat.cpp:828).
struct ColRow {
	const char* id; uint32_t idl;          // read ID, already cut (appendReadID aln_sink.h:2202-2217)
	const char* sid; uint32_t sl;          // seqID
	const char* rank; uint32_t rl;         // taxRank
	const char* name; uint32_t nl;         // taxName ("" when the name table has no entry)
	uint64_t taxid, score, sec, hitlen, qlen, num;
	const uint8_t* seq[2]; uint32_t len[2];
	const char* qual[2]; uint32_t qn[2];
	bool paired;
};

CFC_HD uint32_t col_digits(uint64_t v) { uint32_t n = 1; while(v >= 10) { v /= 10; n++; } return n; }

template <class O> CFC_HD void col_qual(O& o, const ColRow& r, int m) { if(r.qual[m]) o.copy(r.qual[m], r.qn[m]); else o.fill('I', r.qn[m]); }

// One row: the fields of `cols`, tab-separated, then a line end.  O is a byte sink with put / copy / fill / bases / num.
template <class O> CFC_HD void emit_row(O& o, const uint8_t* cols, uint32_t n, const ColRow& r) {
	for(uint32_t i = 0; i < n; i++) {
		if(i) o.put('\t');
		switch(cols[i]) {
			case COL_READ_ID: o.copy(r.id, r.idl); break;
			case COL_SEQ_ID: o.copy(r.sid, r.sl); break;
			case COL_SEQ: o.bases(r.seq[0], r.len[0]); if(r.paired) { o.put('_'); o.bases(r.seq[1], r.len[1]); } break;
			case COL_QUAL: col_qual(o, r, 0); if(r.paired) { o.put('_'); col_qual(o, r, 1); } break;
			case COL_SEQ1: o.bases(r.seq[0], r.len[0]); break;
			case COL_QUAL1: col_qual(o, r, 0); break;
			case COL_SEQ2: if(r.paired) o.bases(r.seq[1], r.len[1]); break;
			case COL_QUAL2: if(r.paired) col_qual(o, r, 1); break;
			case COL_TAX_ID: o.num(r.taxid & 0xffffffffull); if(r.taxid >> 32) { o.put('.'); o.num(r.taxid >> 32); } break;   // appendTaxID :2237-2250
			case COL_TAX_RANK: o.copy(r.rank, r.rl); break;
			case COL_TAX_NAME: o.copy(r.name, r.nl); break;
			case COL_SCORE: o.num(r.score); break;
			case COL_SCORE2: o.num(r.sec); break;
			case COL_HIT_LENGTH: o.num(r.hitlen); break;
			case COL_QUERY_LENGTH: o.num(r.qlen); break;
			case COL_NUM_MATCHES: o.num(r.num); break;
			case COL_PLACEHOLDER: case COL_PLACEHOLDER_STAR: o.put('*'); o.put('0'); break;   // the reference's cases fall through: "" "*" "0"
			case COL_PLACEHOLDER_ZERO: o.put('0'); break;
			default: break;
		}
	}
	o.put('\n');
}

// byte sinks every caller can use: a counter (row sizes) and a one-thread writer
struct ColCount {
	uint64_t n = 0;
	CFC_HD void put(char) { n++; }
	CFC_HD void copy(const char*, uint32_t k) { n += k; }
	CFC_HD void fill(char, uint32_t k) { n += k; }
	CFC_HD void bases(const uint8_t*, uint32_t k) { n += k; }
	CFC_HD void num(uint64_t v) { n += col_digits(v); }
};
struct ColWriter {
	char* p;
	CFC_HD void put(char c) { *p++ = c; }
	CFC_HD void copy(const char* s, uint32_t k) { for(uint32_t i = 0; i < k; i++) p[i] = s[i]; p += k; }
	CFC_HD void fill(char c, uint32_t k) { for(uint32_t i = 0; i < k; i++) p[i] = c; p += k; }
	CFC_HD void bases(const uint8_t* b, uint32_t k) { for(uint32_t i = 0; i < k; i++) p[i] = "ACGTN"[b[i]]; p += k; }
	CFC_HD void num(uint64_t v) { char t[20]; int n = 0; do { t[n++] = (char)('0' + v % 10); v /= 10; } while(v); while(n) *p++ = t[--n]; }
};

}  // namespace cfb

#endif  // CF_COLS_H_
