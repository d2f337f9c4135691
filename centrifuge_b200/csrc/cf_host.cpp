// cf_host.cpp -- host worker around the C ABI: the part of `centrifuge-class` that stays on the CPU.
//
// Replaces (paths relative to the reference tree):
//   option handling of the classification-relevant flags          centrifuge.cpp:530-695,1495
//   PatternSource FASTA/FASTQ parsing + per-read seed              pat.cpp:725-1157, pat.h:55-91
//   quality encodings (--phred64, --solexa-quals, --int-quals)      qual.h:105-171, pat.cpp:997-1078 (cf_quals.h)
//   per-read filters (N ceiling --n-ceil, length >= 2)             centrifuge.cpp:2550-2596, scoring.cpp:104-168
//   AlnSinkWrap::finishRead -> selectByScore -> TSV row            aln_sink.h:1634-1927,2202-2361
//   SpeciesMetrics + SQUAREM abundance + report TSV                aln_sink.h:56-495, centrifuge.cpp:3231-3319
// The classification itself (Classifier::go) happens on the GPU through cfb_classify_submit/wait;
// reads are cut into batches, two batches are in flight, and output order is input order
// (what the reference produces with -p 1 or --reorder).
#include "../../include/cfb200.h"
#include "cf_index.h"
#include "cf_cols.h"
#include "cf_nceil.h"
#include "cf_quals.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <limits>
#include <map>
#include <set>
#include <sstream>
#include <string>
#include <unordered_map>
#include <vector>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

using namespace cfb;

// the loader's HostIndex lives inside cfb_index; the driver only needs these accessors
extern "C" const cfb::HostIndex* cfb_index_host(const cfb_index*);
extern "C" int cfb_device_count(void);

namespace {

struct Options {
	std::string index, out = "-", report = "centrifuge_report.tsv";
	std::vector<std::string> singles, mates1, mates2;
	bool fasta = false, abundance = true, quiet = false, time = false;
	int device = 0; std::vector<int> devices;      // --device N / --devices 0-7: reads are dealt round-robin to the listed GPUs (index replicated)
	uint64_t skip = 0, upto = std::numeric_limits<uint64_t>::max();
	uint32_t seed = 0;
	size_t batch_units = 1u << 18;
	size_t text_block = 64u << 20;      // bytes of read file per device span (text operator)
	bool host_parse = false;            // force the host reader / formatter
	bool separator = false;             // --separator: a report and a separator line after every input (end_input)
	std::string kreport; bool kr_zeros = false, kr_has_score = false, kr_has_len = false; long long kr_min_score = 0, kr_min_len = 0;
	cfb_params prm; std::vector<uint64_t> host, excl;
	int trim5 = 0, trim3 = 0;
	ColList cols;                       // --tab-fmt-cols (the reference's default list unless given)
	NCeil nceil;                        // --n-ceil (L,0,0.15 unless given)
	Quals quals;                        // --phred64 / --solexa-quals / --int-quals (phred33 unless given)
	int kr_col[4] = {0, 2, 3, 5};       // columns the Kraken-style report reads: readID, taxID, score, hitLength
	Options() { std::string e; cols.parse(kDefaultCols, e); }
	bool keep_qual() const { return (cols.mask() & kColQualBits) != 0; }
};

struct OptDesc { const char* name; int has_arg; };
static const OptDesc kLong[] = {
	{"quiet", 0}, {"time", 0}, {"seed", 1}, {"upto", 1}, {"qupto", 1}, {"skip", 1}, {"version", 0}, {"help", 0}, {"threads", 1},
	{"reorder", 0}, {"mm", 0}, {"wrapper", 1}, {"arg-desc", 0}, {"report-file", 1}, {"no-abundance", 0}, {"no-traverse", 0},
	{"min-hitlen", 1}, {"host-taxids", 1}, {"exclude-taxids", 1}, {"classification-rank", 1}, {"trim5", 1}, {"trim3", 1},
	{"device", 1}, {"devices", 1}, {"batch-units", 1}, {"text-block-mb", 1}, {"host-parse", 0},
	{"kreport-file", 1}, {"kreport-show-zeros", 0}, {"kreport-min-score", 1}, {"kreport-min-length", 1},
	{"tab-fmt-cols", 1}, {"passthrough", 0}, {"separator", 0},
	{"n-ceil", 1}, {"ignore-quals", 0}, {"nofw", 0}, {"norc", 0},
	{"phred33", 0}, {"phred33-quals", 0}, {"phred64", 0}, {"phred64-quals", 0}, {"solexa1.3-quals", 0}, {"solexa-quals", 0},
	{"int-quals", 0}, {"integer-quals", 0}, {NULL, 0}};
static const char* kShort = "fqtu:s:p:k:1:2:U:x:S:3:5:h";

std::vector<std::string> split(const std::string& s, char d) {
	std::vector<std::string> v; std::string t; std::stringstream ss(s);
	while(std::getline(ss, t, d)) if(!t.empty()) v.push_back(t);
	return v;
}

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// ------------------------------------------------------------------------------ compressed input
// A regular file that starts with 1f 8b 08 is gzip, one that starts with "BZh" + a level digit + a block or
// end-of-stream magic is bzip2: its bytes are decompressed on the device (cfb_gunzip_* / cfb_bunzip2_*, on the first
// listed device) and everything downstream sees the decompressed bytes.  FIFOs and stdin are read as they are.
static int g_gz_device = 0;
struct GzTotals { uint64_t files = 0, st[6] = {0, 0, 0, 0, 0, 0}; double t = 0; };
static GzTotals g_gz, g_bz;                     // per format: gzip, bzip2
// One input file (or pair) of the command line can be read twice: in spans, then by the record-level reader from a
// span that failed.  Its trailing-garbage warning is printed once per such input, keyed by its position in the list.
static std::atomic<uint64_t> g_input_seq(0);
static std::mutex g_warn_mu;
static std::set<std::pair<uint64_t, std::string>> g_warned;

enum { FMT_PLAIN = 0, FMT_GZIP = 1, FMT_BZIP2 = 2 };
static int compressed_format(int fd) {
	unsigned char m[10];
	const ssize_t k = pread(fd, m, 10, 0);
	if(k >= 3 && m[0] == 0x1f && m[1] == 0x8b && m[2] == 8) return FMT_GZIP;
	static const unsigned char blk[6] = {0x31, 0x41, 0x59, 0x26, 0x53, 0x59}, eos[6] = {0x17, 0x72, 0x45, 0x38, 0x50, 0x90};
	if(k == 10 && m[0] == 'B' && m[1] == 'Z' && m[2] == 'h' && m[3] >= '1' && m[3] <= '9' && (!memcmp(m + 4, blk, 6) || !memcmp(m + 4, eos, 6)))
		return FMT_BZIP2;
	return FMT_PLAIN;
}

struct GzReader {        // decompressed bytes of one gzip or bzip2 file
	std::string path; int fd = -1; cfb_gunzip* g = NULL; cfb_bunzip2* bz = NULL;
	std::vector<unsigned char> in; size_t in_lo = 0, in_hi = 0; uint64_t file_off = 0; bool file_eof = false;
	std::vector<unsigned char> look; size_t look_lo = 0, look_hi = 0;       // read-ahead for peek()
	bool done = false, starved = false; double t = 0;
	std::string err;                                                        // "Error: <file>: <reason>" once something failed
	bool open(const std::string& p, int fd_, int fmt) {
		path = p; fd = fd_;
		const int rc = fmt == FMT_BZIP2 ? cfb_bunzip2_create(g_gz_device, 0, &bz) : cfb_gunzip_create(g_gz_device, 0, &g);
		if(rc != CFB_OK) { err = "Error: " + path + ": " + cfb_last_error(); return false; }
		in.resize(64u << 20);
		return true;
	}
	void close() {
		if(g) {
			uint64_t st[5]; cfb_gunzip_stats(g, st);
			g_gz.files++; for(int k = 0; k < 5; k++) g_gz.st[k] += st[k]; g_gz.t += t;
			cfb_gunzip_destroy(g); g = NULL;
		}
		if(bz) {
			uint64_t st[6]; cfb_bunzip2_stats(bz, st);
			g_bz.files++; for(int k = 0; k < 6; k++) g_bz.st[k] += st[k]; g_bz.t += t;
			if(st[5] && err.empty()) {
				std::lock_guard<std::mutex> lk(g_warn_mu);
				if(g_warned.insert(std::make_pair(g_input_seq.load(), path)).second)
					std::cerr << "Warning: " << path << ": trailing garbage after the last bzip2 stream ignored" << std::endl;
			}
			cfb_bunzip2_destroy(bz); bz = NULL;
		}
		if(fd >= 0) ::close(fd);
		fd = -1;
	}
	size_t raw_read(unsigned char* dst, size_t n) {
		size_t got = 0;
		while(got < n && !done && err.empty()) {
			if(!file_eof && (in_hi - in_lo < in.size() / 2 || starved)) {
				starved = false;
				memmove(in.data(), in.data() + in_lo, in_hi - in_lo); in_hi -= in_lo; in_lo = 0;
				while(in_hi < in.size()) {
					const ssize_t r = pread(fd, in.data() + in_hi, in.size() - in_hi, (off_t)file_off);
					if(r < 0) { err = "Error: " + path + ": read failed"; return got; }
					if(r == 0) { file_eof = true; break; }
					in_hi += (size_t)r; file_off += (uint64_t)r;
				}
			}
			uint64_t no = 0, nc = 0;
			const double t0 = now_s();
			const int rc = bz ? cfb_bunzip2_run(bz, in.data() + in_lo, in_hi - in_lo, file_eof ? 1 : 0, dst + got, n - got, &no, &nc)
			                  : cfb_gunzip_run(g, in.data() + in_lo, in_hi - in_lo, file_eof ? 1 : 0, dst + got, n - got, &no, &nc);
			t += now_s() - t0;
			if(rc != CFB_OK) { err = "Error: " + path + ": " + cfb_last_error(); return got; }
			in_lo += nc; got += no;
			if(no == 0 && nc == 0) {
				if(file_eof) done = true;
				else {                                      // the decoder needs more than it was given: read more before the next call
					if(in_hi - in_lo == in.size()) in.resize(in.size() * 2);
					starved = true;
				}
			}
		}
		return got;
	}
	size_t read(unsigned char* dst, size_t n) {
		size_t got = std::min(n, look_hi - look_lo);
		memcpy(dst, look.data() + look_lo, got); look_lo += got;
		return got + raw_read(dst + got, n - got);
	}
	int peek() {
		if(look_lo == look_hi) {
			look.resize(1 << 16); look_lo = 0;
			look_hi = raw_read(look.data(), look.size());
		}
		return look_lo < look_hi ? look[look_lo] : -1;
	}
};

// ------------------------------------------------------------------------------ reads
struct FileIn {       // buffered byte source with one-byte peek
	FILE* f = NULL; std::vector<unsigned char> buf; size_t pos = 0, end = 0;
	GzReader* gz = NULL; std::string path;
	bool open(const std::string& p) {
		path = p; buf.resize(1 << 22);
		if(p != "-") {
			struct stat st;
			if(::stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode)) {
				const int fd = ::open(p.c_str(), O_RDONLY);
				const int fmt = fd >= 0 ? compressed_format(fd) : FMT_PLAIN;
				if(fmt != FMT_PLAIN) {
					gz = new GzReader();
					if(!gz->open(p, fd, fmt)) { std::cerr << gz->err << std::endl; throw 1; }
					return true;
				}
				if(fd >= 0) ::close(fd);
			}
		}
		f = p == "-" ? stdin : fopen(p.c_str(), "rb"); return f != NULL;
	}
	// gzip / bzip2: decompress again from the start of the file and drop the first `off` decompressed bytes
	bool seek(uint64_t off) {
		pos = end = 0;
		if(gz) {
			std::vector<unsigned char> skip(1 << 22);
			while(off) { const size_t r = gz->read(skip.data(), (size_t)std::min<uint64_t>(off, skip.size())); if(!gz->err.empty()) { std::cerr << gz->err << std::endl; throw 1; } if(!r) return false; off -= r; }
			return true;
		}
		return f && f != stdin && fseeko(f, (off_t)off, SEEK_SET) == 0;
	}
	void close() { if(gz) { gz->close(); delete gz; gz = NULL; } if(f && f != stdin) fclose(f); f = NULL; }
	inline bool fill() {
		if(gz) { end = gz->read(buf.data(), buf.size()); pos = 0; if(!gz->err.empty()) { std::cerr << gz->err << std::endl; throw 1; } return end > 0; }
		if(!f) return false;
		end = fread(buf.data(), 1, buf.size(), f); pos = 0; return end > 0;
	}
	inline int get() { if(pos == end && !fill()) return -1; return buf[pos++]; }
	inline int peek() { if(pos == end && !fill()) return -1; return buf[pos]; }
};

static uint8_t g_asc2dna[256];
static uint8_t g_dnacat[256];
static void init_tables() {
	static bool done = false; if(done) return; done = true;
	memset(g_asc2dna, 0, 256); memset(g_dnacat, 0, 256);
	g_asc2dna['C'] = g_asc2dna['c'] = 1; g_asc2dna['G'] = g_asc2dna['g'] = 2; g_asc2dna['T'] = g_asc2dna['t'] = 3; g_asc2dna['N'] = g_asc2dna['n'] = 4;
	const char* k = "ABCDGHKMNRSTVWXY";                  // asc2dnacat > 0 (alphabet.cpp:36-58) plus '-'
	for(const char* p = k; *p; p++) { g_dnacat[(int)*p] = 1; g_dnacat[tolower(*p)] = 1; }
	g_dnacat['-'] = 1;
}

struct Rec {          // one parsed read
	std::string name; std::vector<uint8_t> seq; uint32_t qx = 0;   // qx = quality contribution to the seed
	std::string qual;     // kept FASTQ qualities, filled only when a quality column is printed
	bool ok = false;
};

// FASTA record, pat.cpp:725-849.  Returns false at end of input.
static bool parse_fasta(FileIn& in, Rec& r, uint64_t& count, bool& first, int trim5, int trim3) {
	r.name.clear(); r.seq.clear(); r.qx = 0;
	int c = in.get();
	if(c < 0) return false;
	while(c == '#' || c == ';' || c == '\r' || c == '\n') {
		// FileBuf::peekUptoNewline (filebuf.h:306-318): drop the rest of the line the cursor is in, then every line end.
		// For a comment that is the comment line; after a *line end* (only possible before the first record) it is
		// the whole next line -- a leading blank line makes the reference swallow the first header (pat.cpp:744-748).
		for(;;) { int d = in.peek(); if(d < 0 || d == '\n' || d == '\r') break; in.get(); }
		while(in.peek() == '\n' || in.peek() == '\r') in.get();
		c = in.get();
		if(c < 0 && !first) return false;
		if(c < 0) break;
	}
	if(first) { if(c != '>') { std::cerr << "Error: reads file does not look like a FASTA file" << std::endl; throw 1; } first = false; }
	c = in.get();
	for(;;) {
		if(c < 0) return false;
		if(c == '\n' || c == '\r') {
			while(c == '\n' || c == '\r') { if(in.peek() == '>') break; c = in.get(); if(c < 0) return false; }
			break;
		}
		r.name.push_back((char)c);
		if(in.peek() == '>') break;
		c = in.get();
	}
	int begin = 0;
	if(!((c == '\n' || c == '\r') && in.peek() == '>')) {
		while(c != '>' && c >= 0) {
			if(g_dnacat[c] && begin++ >= trim5) r.seq.push_back(g_asc2dna[c]);
			if(in.peek() == '>') break;
			c = in.get();
		}
	}
	if(trim3 > 0) r.seq.resize(r.seq.size() > (size_t)trim3 ? r.seq.size() - trim3 : 0);
	// quality of every FASTA base is 'I' (pat.cpp:828): fold into the seed contribution
	for(size_t i = 0; i < r.seq.size(); i++) r.qx ^= ((uint32_t)'I' << ((i & 3) << 3));
	if(r.name.empty()) { char b[32]; snprintf(b, sizeof b, "%llu", (unsigned long long)count); r.name = b; }
	count++;
	return true;
}

static const uint32_t g_sol_steps = solexa_steps();      // the Solexa -> Phred table (cf_quals.h)

// Integer qualities of one record, pat.cpp:997-1030: the line as FileBuf::gets(buf, 4096) takes it (at most 4095 bytes;
// the byte after them is consumed and dropped, the rest of a longer line stays in the stream, and string(buf) ends at a
// NUL), split on ' ' as tokenize does (a leading space gives an empty first token, runs and trailing spaces none), each
// token through atoi and intToPhred33 -- every token, trimmed ones included -- then the kept ones from trim5 on, minus
// trim3, must cover the read and may be one longer; the string is cut to the read's length.
static void parse_int_quals(FileIn& in, Rec& r, int trim5, int trim3, const Quals& qe, std::string& q) {
	std::string line;
	size_t stored = 0;
	for(;;) {
		const int d = in.get();
		if(d < 0) break;
		if(stored == 4095 || d == '\n' || d == '\r') { while(in.peek() == '\n' || in.peek() == '\r') in.get(); break; }
		line.push_back((char)d); stored++;
	}
	if(stored) {                                           // tokenizeQualLine returns no tokens for an empty line
		const std::string s(line.c_str());
		size_t last = 0, pos = s.find(' ');
		int j = 0;
		while(pos != std::string::npos || last != std::string::npos) {
			const size_t e = pos == std::string::npos ? s.size() : pos;
			const int pq = qual_from_int(qual_atoi(s.data() + last, s.data() + e), qe.solexa, g_sol_steps);
			if(pq < 33) { std::cerr << qual_int_error(pq) << std::endl; throw 1; }
			if(j++ >= trim5) q.push_back((char)pq);
			last = s.find_first_not_of(' ', pos);
			pos = s.find(' ', last);
		}
	}
	q.resize(q.size() > (size_t)trim3 ? q.size() - trim3 : 0);
	if(q.size() < r.seq.size()) { std::cerr << "Error: Read " << r.name << " has more read characters than quality values." << std::endl; throw 1; }
	if(q.size() > r.seq.size() + 1) { std::cerr << "Error: Read " << r.name << " has more quality values than read characters." << std::endl; throw 1; }
	q.resize(r.seq.size());
}

// FASTQ record, pat.cpp:852-1157 (no colour/fuzzy modes), qualities in the encoding `qe` converted to phred33.
static bool parse_fastq(FileIn& in, Rec& r, uint64_t& count, bool& first, int trim5, int trim3, bool keep_qual = false, const Quals& qe = Quals()) {
	r.name.clear(); r.seq.clear(); r.qual.clear(); r.qx = 0;
	int c;
	if(first) {
		c = in.get();
		while(c == '\n' || c == '\r') c = in.get();
		if(c < 0) return false;
		if(c != '@') { std::cerr << "Error: reads file does not look like a FASTQ file" << std::endl; throw 1; }
		first = false;
	}
	for(;;) {
		c = in.get();
		if(c < 0) return false;
		if(c == '\n' || c == '\r') { while(c == '\n' || c == '\r') { c = in.get(); if(c < 0) return false; } break; }
		r.name.push_back((char)c);
	}
	int nread = 0;
	while(c != '+') {
		if(c == '.') c = 'N';
		if(isalpha(c)) { if(nread >= trim5) r.seq.push_back(g_asc2dna[c]); nread++; }
		c = in.get();
		if(c < 0) return false;
	}
	if(trim3 > 0) r.seq.resize(r.seq.size() > (size_t)trim3 ? r.seq.size() - trim3 : 0);
	for(;;) { int d = in.get(); if(d < 0) break; if(d == '\n' || d == '\r') { while(in.peek() == '\n' || in.peek() == '\r') in.get(); break; } }
	if(nread == 0) { if(in.peek() == '@') in.get(); count++; return true; }
	if(qe.integer) {
		std::string q;
		parse_int_quals(in, r, trim5, trim3, qe, q);
		for(size_t i = 0; i < q.size(); i++) r.qx ^= (uint32_t)(int32_t)(int8_t)q[i] << ((i & 3) << 3);   // chars are signed in genRandSeed
		if(keep_qual) r.qual.swap(q);
	} else {
		// character qualities: pat.cpp:1042-1078.  Everything from trim5 on is kept and converted (charToPhred33), then
		// trim3 is cut off the end; the kept string must be as long as the read or one longer.  A space anywhere is refused.
		size_t qn = 0, kept = 0; int qi = 0;
		for(;;) {
			c = in.get();
			if(c == ' ') {
				std::cerr << "Error: Encountered one or more spaces while parsing the quality string for read " << r.name << ".  If this is a FASTQ file with integer (non-ASCII-encoded) qualities, try re-running with the --integer-quals option." << std::endl;
				throw 1;
			}
			if(c < 0 || c == '\r' || c == '\n') break;
			if(qi >= trim5) {
				const int q = qual_from_char((uint32_t)c, qe.solexa, qe.phred64, g_sol_steps);
				if(q < 0) { std::cerr << qual_char_error((uint32_t)c, qe.phred64) << std::endl; throw 1; }
				kept++;
				if(keep_qual) r.qual.push_back((char)q);
				if(qn < r.seq.size()) { r.qx ^= (uint32_t)(int32_t)(int8_t)q << ((qn & 3) << 3); qn++; }
			}
			qi++;
		}
		kept = kept > (size_t)trim3 ? kept - trim3 : 0;
		if(keep_qual) r.qual.resize(kept);
		if(kept < r.seq.size()) { std::cerr << "Error: Read " << r.name << " has more read characters than quality values." << std::endl; throw 1; }
		if(kept > r.seq.size() + 1) { std::cerr << "Error: Read " << r.name << " has more quality values than read characters." << std::endl; throw 1; }
	}
	while(in.peek() == '\n' || in.peek() == '\r') in.get();
	in.get();                                              // '@' of the next record (or EOF)
	if(r.name.empty()) { char b[32]; snprintf(b, sizeof b, "%llu", (unsigned long long)count); r.name = b; }
	count++;
	return true;
}

static uint32_t read_seed(const Rec& r, uint32_t seed) {   // genRandSeed pat.h:55-91
	uint32_t rseed = (seed + 101) * 59 * 61 * 67 * 71 * 73 * 79 * 83;
	const size_t n = r.seq.size();
	for(size_t i = 0; i < n; i++) rseed ^= ((uint32_t)r.seq[i] << ((i & 15) << 1));
	rseed ^= r.qx;
	for(size_t i = 0; i < r.name.size(); i++) { const int p = (int)r.name[i]; if(p == '/') break; rseed ^= ((uint32_t)p << ((i & 3) << 3)); }
	return rseed;
}
static bool passes_filters(const std::vector<uint8_t>& s, const NCeil& f) {   // nFilter (--n-ceil) + lenfilt
	return nceil_filter(f, s.data(), s.size());
}

struct HostBatch {     // one batch staged for the GPU plus what the formatter needs afterwards
	std::vector<uint8_t> bases; std::vector<uint64_t> off[2]; std::vector<uint32_t> len[2]; std::vector<uint8_t> flags;
	std::vector<uint32_t> seedA, seedB; std::vector<char> names; std::vector<uint32_t> name_off;
	std::vector<char> quals; std::vector<uint64_t> qoff[2]; std::vector<uint32_t> qn[2];   // kept FASTQ qualities, only with a quality column (qual_mode 1)
	bool paired = false; size_t n = 0; int qual_mode = 0;       // 0: no quality column, 1: FASTQ, 2: FASTA (all 'I')
	void clear(bool p) { bases.clear(); for(int m = 0; m < 2; m++) { off[m].clear(); len[m].clear(); qoff[m].clear(); qn[m].clear(); } flags.clear(); seedA.clear(); seedB.clear(); names.clear(); name_off.clear(); quals.clear(); paired = p; n = 0; }
	void add_qual(int m, const Rec& r) { if(qual_mode != 1) return; qoff[m].push_back(quals.size()); qn[m].push_back((uint32_t)r.qual.size()); quals.insert(quals.end(), r.qual.begin(), r.qual.end()); }
	void add(const Rec& a, const Rec* b, uint32_t seed, const NCeil& nc) {
		add_qual(0, a); if(paired) add_qual(1, *b);
		off[0].push_back(bases.size()); len[0].push_back((uint32_t)a.seq.size()); bases.insert(bases.end(), a.seq.begin(), a.seq.end());
		uint8_t fl = passes_filters(a.seq, nc) ? 1 : 0;
		seedA.push_back(read_seed(a, seed));
		if(paired) {
			off[1].push_back(bases.size()); len[1].push_back((uint32_t)b->seq.size()); bases.insert(bases.end(), b->seq.begin(), b->seq.end());
			if(!b->seq.empty() && passes_filters(b->seq, nc)) fl |= 2;
			seedB.push_back(b->seq.empty() ? 0u : read_seed(*b, seed));
		}
		flags.push_back(fl);
		name_off.push_back((uint32_t)names.size()); names.insert(names.end(), a.name.begin(), a.name.end());
		n++;
	}
};

// ------------------------------------------------------------------------------ metrics
struct IdsLess {       // SpeciesMetrics::IDs::operator< aln_sink.h:63-71
	bool operator()(const std::vector<uint64_t>& a, const std::vector<uint64_t>& b) const {
		if(a.size() != b.size()) return a.size() < b.size();
		for(size_t i = 0; i < a.size(); i++) if(a[i] != b[i]) return a[i] < b[i];
		return false;
	}
};
struct Counts { uint64_t n_reads = 0, n_unique = 0; };
struct Species {
	std::map<uint64_t, Counts> counts;
	std::map<std::vector<uint64_t>, uint64_t, IdsLess> observed;
	std::vector<uint64_t> cur;
	std::map<uint64_t, double> abundance_len;
	uint64_t last_tax = ~0ull; Counts* last = NULL;
	void reset_counts() { counts.clear(); last = NULL; }       // SpeciesMetrics::reset aln_sink.h:84-91: `observed` stays
	inline void add(uint64_t taxid, int64_t score, int64_t max_score, uint32_t nresult) {   // addSpeciesCounts aln_sink.h:142-172
		if(taxid != last_tax || !last) { last = &counts[taxid]; last_tax = taxid; }
		last->n_reads++; if(nresult == 1) last->n_unique++;
		if(score >= max_score) {
			cur.push_back(taxid);
			if(cur.size() == nresult) { std::sort(cur.begin(), cur.end()); observed[cur] += 1; cur.clear(); }
		}
	}
};

typedef std::map<std::vector<uint64_t>, uint64_t, IdsLess> Observed;

// The EM works on a flattened copy of `observed`: for every key, in map order, the species slots its ids
// contribute to, in the order the reference's nested loops visit them (aln_sink.h:196-272: the id itself when it
// is a leaf slot, else its leaf descendants in ascending taxid).  Sums run in that order, so every double is the
// reference's.  The same arrays drive the device version (cfb_em_abundance, SURVEY.md 8f rank 3).
struct EmFlat {
	std::vector<uint64_t> count; std::vector<uint64_t> key_off; std::vector<uint32_t> target;   // K, K+1, T
	std::vector<uint64_t> len;                                                                    // n
};
static void em_step(const EmFlat& f, const std::vector<double>& p, std::vector<double>& pn) {   // aln_sink.h:196-272
	std::fill(pn.begin(), pn.end(), 0.0);
	const size_t K = f.count.size();
	for(size_t k = 0; k < K; k++) {
		double psum = 0.0;
		for(uint64_t t = f.key_off[k]; t < f.key_off[k + 1]; t++) psum += p[f.target[t]];
		if(psum == 0.0) continue;
		const uint64_t count = f.count[k];
		for(uint64_t t = f.key_off[k]; t < f.key_off[k + 1]; t++) { const uint32_t j = f.target[t]; pn[j] += (count * (p[j] / psum)); }
	}
	double sum = 0.0;
	for(size_t i = 0; i < pn.size(); i++) sum += (pn[i] / f.len[i]);
	for(size_t i = 0; i < pn.size(); i++) pn[i] = pn[i] / f.len[i] / sum;
}

// SQUAREM-accelerated iteration on the host (aln_sink.h:410-480): same loop the device version restates
static void em_iterate(const EmFlat& f, std::vector<double>& p, size_t& it, double& diff) {
	std::vector<double> pn(p.size()), pn2(p.size()), pr(p.size()), pv(p.size());
	it = 0; diff = 0.0;
	for(;;) {
		em_step(f, p, pn);
		em_step(f, pn, pn2);
		double ssr = 0.0, ssv = 0.0;
		for(size_t i = 0; i < p.size(); i++) { pr[i] = pn[i] - p[i]; ssr += pr[i] * pr[i]; pv[i] = pn2[i] - pn[i] - pr[i]; ssv += pv[i] * pv[i]; }
		if(ssv > 0.0) {
			const double g = -sqrt(ssr / ssv);
			for(size_t i = 0; i < p.size(); i++) pn2[i] = std::max(0.0, p[i] - 2 * g * pr[i] + g * g * pv[i]);
			em_step(f, pn2, pn);
		}
		diff = 0.0;
		for(size_t i = 0; i < p.size(); i++) diff += (p[i] > pn[i] ? p[i] - pn[i] : pn[i] - p[i]);
		if(diff < 0.0000000001) break;
		if(++it >= 10000) break;
		p = pn;
	}
}

extern "C" int cfb_em_abundance(int device, uint64_t n, uint64_t K, const uint64_t* count, const uint64_t* key_off, const uint32_t* target,
                                const uint64_t* len, double* p, uint64_t* iters, double* last_diff);
extern "C" const char* cfb_em_last_error(void);

static void calc_abundance(const HostIndex& h, Species& sp, size_t& iters, double& last_diff, int device) {   // aln_sink.h:274-495
	std::set<uint64_t> leaves;
	for(Observed::const_iterator it = sp.observed.begin(); it != sp.observed.end(); ++it)
		for(size_t i = 0; i < it->first.size(); i++) { const TaxNode* n = h.find_node(it->first[i]); if(n && n->leaf) leaves.insert(n->taxid); }
	std::map<uint64_t, std::vector<uint64_t> > anc;
	for(Observed::const_iterator it = sp.observed.begin(); it != sp.observed.end(); ++it)
		for(size_t i = 0; i < it->first.size(); i++) {
			const uint64_t tid = it->first[i];
			if(leaves.count(tid) || anc.count(tid)) continue;
			std::vector<uint64_t>& ch = anc[tid];
			for(std::set<uint64_t>::const_iterator l = leaves.begin(); l != leaves.end(); ++l) {
				for(uint64_t t = *l;;) {
					const TaxNode* n = h.find_node(t);
					if(!n) break;
					if(tid == n->parent) ch.push_back(*l);
					if(t == n->parent) break;
					t = n->parent;
				}
			}
			std::sort(ch.begin(), ch.end());
		}
	std::map<uint64_t, uint64_t> t2n; std::vector<double> p; EmFlat f;
	for(Observed::const_iterator it = sp.observed.begin(); it != sp.observed.end(); ++it) {
		const std::vector<uint64_t>& ids = it->first; const uint64_t count = it->second;
		for(size_t i = 0; i < ids.size(); i++) {
			const uint64_t tid = ids[i];
			if(!leaves.count(tid)) continue;
			std::map<uint64_t, uint64_t>::iterator fnd = t2n.find(tid);
			if(fnd == t2n.end()) {
				t2n[tid] = p.size(); p.push_back(1.0 / ids.size() * count);
				std::map<uint64_t, uint64_t>::const_iterator s = h.sizes.find(tid);
				f.len.push_back(s != h.sizes.end() ? s->second : (uint64_t)std::numeric_limits<size_t>::max());
			} else p[fnd->second] += (1.0 / ids.size() * count);
		}
	}
	{ double sum = 0.0; for(size_t i = 0; i < p.size(); i++) sum += (p[i] / f.len[i]); for(size_t i = 0; i < p.size(); i++) p[i] = (p[i] / f.len[i]) / sum; }
	f.key_off.push_back(0);
	for(Observed::const_iterator it = sp.observed.begin(); it != sp.observed.end(); ++it) {
		const std::vector<uint64_t>& ids = it->first;
		for(size_t i = 0; i < ids.size(); i++) {
			std::map<uint64_t, uint64_t>::const_iterator id = t2n.find(ids[i]);
			if(id != t2n.end()) { f.target.push_back((uint32_t)id->second); continue; }
			std::map<uint64_t, std::vector<uint64_t> >::const_iterator a = anc.find(ids[i]);
			if(a == anc.end()) continue;
			for(size_t c = 0; c < a->second.size(); c++) { std::map<uint64_t, uint64_t>::const_iterator ci = t2n.find(a->second[c]); if(ci != t2n.end()) f.target.push_back((uint32_t)ci->second); }
		}
		f.count.push_back(it->second); f.key_off.push_back(f.target.size());
	}
	// large problems (or CFB_GPU_EM=1) iterate on the device: same operations in the same order, same doubles
	const char* ge = getenv("CFB_GPU_EM");
	const bool on_device = device >= 0 && !p.empty() && ((ge && ge[0] == '1') || (!(ge && ge[0] == '0') && f.target.size() >= (1u << 18)));
	if(getenv("CFB_TEXT_STATS"))
		std::cerr << "[cfb] abundance EM: " << p.size() << " species, " << f.count.size() << " keys, " << f.target.size() << " contributions, on the "
		          << (on_device ? "device" : "host") << std::endl;
	size_t it = 0; double diff = 0.0;
	if(on_device) {
		uint64_t iters64 = 0;
		if(cfb_em_abundance(device, p.size(), f.count.size(), f.count.data(), f.key_off.data(), f.target.data(), f.len.data(), p.data(), &iters64, &diff) != CFB_OK) {
			std::cerr << "Error: " << cfb_em_last_error() << std::endl; throw 1;
		}
		it = (size_t)iters64;
	} else em_iterate(f, p, it, diff);
	iters = it; last_diff = diff;
	sp.abundance_len.clear();
	for(std::map<uint64_t, uint64_t>::iterator i = t2n.begin(); i != t2n.end(); ++i) sp.abundance_len[i->first] = p[i->second];
}

// ------------------------------------------------------------------------------ formatting
struct Lcg {           // RandomSource random_source.h:34-61
	uint32_t last;
	inline uint32_t next() { last = 1664525u * last + 1013904223u; uint32_t r = last >> 16; last = 1664525u * last + 1013904223u; return r ^ last; }
};

struct Formatter {
	const HostIndex& h; const Options& o; Species& sp;
	std::vector<char> out;
	std::vector<std::pair<int64_t, uint32_t> > buf;
	Formatter(const HostIndex& h_, const Options& o_, Species& s) : h(h_), o(o_), sp(s) {}

	void format_batch(const HostBatch& hb, const cfb_result& res) {
		out.clear();
		const uint8_t* cols = o.cols.fields.data(); const uint32_t ncols = (uint32_t)o.cols.fields.size();
		const bool need_name = (o.cols.mask() & (1u << COL_TAX_NAME)) != 0;
		for(size_t u = 0; u < hb.n; u++) {
			const uint32_t r0 = res.rec_off[u], r1 = res.rec_off[u + 1];
			const uint32_t sz = r1 > r0 ? r1 - r0 : 1;
			const bool uncl = r1 == r0;
			const uint8_t fl = hb.flags[u];
			const bool f1 = fl & 1, f2 = (fl & 2) != 0;
			// max score of the mates that were classified (classifier.h:530-535); 0 for "unclassified"
			int64_t max_score = 0;
			if(!uncl) {
				if(f1) { const int64_t L = hb.len[0][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
				if(f2) { const int64_t L = hb.len[1][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
			}
			Lcg rnd; rnd.last = (f1 && f2) ? (hb.seedA[u] ^ hb.seedB[u]) : hb.seedA[u];   // centrifuge.cpp:2609-2613
			// AlnSetSumm::init aligner_result.h:398-427
			const int64_t INV = std::numeric_limits<int64_t>::min();
			int64_t best = INV, sec = INV;
			buf.resize(sz);
			for(uint32_t k = 0; k < sz; k++) {
				const int64_t sc = uncl ? 0 : (int64_t)res.recs[r0 + k].score;
				if(sc > best) { sec = best; best = sc; } else if(sc > sec) sec = sc;
				buf[k] = std::make_pair(sc, k);
			}
			// selectByScore aln_sink.h:1861-1927
			size_t num = std::min<size_t>(sz, (size_t)o.prm.khits);
			if(sz > 1) {
				std::sort(buf.begin(), buf.end()); std::reverse(buf.begin(), buf.end());
				size_t streak = 0;
				for(size_t k = 1; k < sz; k++) {
					if(buf[k].first == buf[k - 1].first) { if(streak == 0) streak = 1; streak++; }
					else { if(streak > 1) shuffle(k - streak, streak, rnd); streak = 0; }
				}
				if(streak > 1) shuffle(sz - streak, streak, rnd);
				for(size_t k = 0; k + 1 < num; k++) if(buf[k].first != buf[k + 1].first) { num = k + 1; break; }
			}
			const char* nm = hb.names.data() + hb.name_off[u];
			size_t nlen = (u + 1 < hb.n ? hb.name_off[u + 1] : hb.names.size()) - hb.name_off[u];
			if(nlen >= 2 && nm[nlen - 2] == '/' && (nm[nlen - 1] == '1' || nm[nlen - 1] == '2' || nm[nlen - 1] == '3')) nlen -= 2;   // appendReadID aln_sink.h:2202
			size_t idlen = 0; while(idlen < nlen && !isspace((unsigned char)nm[idlen])) idlen++;
			ColRow row; memset(&row, 0, sizeof row);
			row.id = nm; row.idl = (uint32_t)idlen; row.paired = hb.paired;
			row.qlen = (uint64_t)hb.len[0][u] + (hb.paired ? hb.len[1][u] : 0);
			row.sec = sec != INV ? (uint64_t)sec : 0; row.num = num;
			for(int m = 0; m < (hb.paired ? 2 : 1); m++) {
				row.seq[m] = hb.bases.data() + hb.off[m][u]; row.len[m] = hb.len[m][u];
				if(hb.qual_mode == 1) { row.qual[m] = hb.quals.data() + hb.qoff[m][u]; row.qn[m] = hb.qn[m][u]; }
				else row.qn[m] = hb.len[m][u];
			}
			for(size_t k = 0; k < num; k++) {
				uint64_t taxid = 0, score = 0, hitlen = 0; uint32_t uid = CFB_UID_NONE;
				if(!uncl) { const cfb_rec& r = res.recs[r0 + buf[k].second]; taxid = r.taxid; score = r.score; hitlen = r.hitlen; uid = r.uid; }
				// seqID: appendSeqID aln_sink.h:2220-2234 on top of the uid chosen at classifier.h:557; taxRank: the node's
				// rank, 0 for unclassified rows (classifier.h:540-546,619-626)
				const char* sid; const char* rk;
				if(uncl) { sid = "unclassified"; rk = rank_name(0); }
				else {
					const TaxNode* n = h.find_node(taxid);
					const bool leaf = n ? n->leaf != 0 : true; const int rank = n ? n->rank : RANK_UNKNOWN;
					rk = rank_name(rank);
					sid = (leaf && uid != CFB_UID_NONE && uid < h.seq_name.size()) ? h.seq_name[uid].c_str() : rk;
				}
				row.sid = sid; row.sl = (uint32_t)strlen(sid); row.rank = rk; row.rl = (uint32_t)strlen(rk);
				row.name = ""; row.nl = 0;
				if(need_name) { std::map<uint64_t, std::string>::const_iterator it = h.names.find(taxid); if(it != h.names.end()) { row.name = it->second.data(); row.nl = (uint32_t)it->second.size(); } }
				row.taxid = taxid; row.score = score; row.hitlen = hitlen;
				ColCount cnt; emit_row(cnt, cols, ncols, row);
				const size_t base = out.size();
				out.resize(base + cnt.n);
				ColWriter w; w.p = out.data() + base; emit_row(w, cols, ncols, row);
				sp.add(taxid, (int64_t)score, max_score, (uint32_t)num);
			}
		}
	}
	inline void shuffle(size_t begin, size_t n, Lcg& rnd) {    // EList::shufflePortion ds.h:784-795
		size_t left = n;
		for(size_t i = begin; i < begin + n - 1; i++) { const uint32_t r = rnd.next() % left; if(r > 0) std::swap(buf[i], buf[i + r]); left--; }
	}
};


// ------------------------------------------------------------------------------ Kraken-style report
// In-process equivalent of the reference's `centrifuge-kreport` script (SURVEY.md 8f rank 4), fed with the
// classification rows while they are still in memory instead of re-reading the TSV.  Same algorithm on the
// same text: rows of one read (equal consecutive readID strings) are merged to their LCA
// (centrifuge-kreport:84-123), clade sums by DFS from node 1 (:219-228), children sorted by clade count,
// stable (:150-156); taxonomy as `centrifuge-inspect --taxonomy-tree/--name-table` prints it
// (centrifuge_inspect.cpp:534-550: ascending taxid).
struct KReport {
	const HostIndex& h; const Options& o;
	std::unordered_map<uint64_t, long long> taxo; long long seq_count = 0;
	std::string prev_id; uint64_t prev_tax = 0; bool have_prev = false;
	std::unordered_map<uint64_t, bool> in_tree_cache;
	uint64_t last_key = ~0ull; long long* last_ctr = NULL;
	KReport(const HostIndex& h_, const Options& o_) : h(h_), o(o_) { taxo[0] = 0; }
	bool enabled() const { return !o.kreport.empty(); }
	bool parent_of(uint64_t t, uint64_t& p) const {          // %parent_map: node 1 hangs under 0
		const TaxNode* n = h.find_node(t);
		if(!n) return false;
		p = t == 1 ? 0 : n->parent;
		return true;
	}
	bool in_tree(uint64_t t) {                                // isTaxIDInTree :160-174
		std::unordered_map<uint64_t, bool>::const_iterator it = in_tree_cache.find(t);
		if(it != in_tree_cache.end()) return it->second;
		bool ok = true;
		for(uint64_t a = t; a > 1;) { uint64_t p; if(!parent_of(a, p)) { std::cerr << "Couldn't find parent of taxID " << a << " - directly assigned to root." << std::endl; ok = false; break; } if(p == a) break; a = p; }
		in_tree_cache[t] = ok;
		return ok;
	}
	uint64_t lca(uint64_t a, uint64_t b) {                    // :176-203
		if(a == 0) return b;
		if(b == 0) return a;
		if(a == b) return a;
		std::set<uint64_t> path;
		while(a >= 1) { path.insert(a); uint64_t p; if(!parent_of(a, p)) break; if(p == a) break; a = p; }
		while(b > 1) { if(path.count(b)) return b; uint64_t p; if(!parent_of(b, p)) break; if(p == b) break; b = p; }
		return 1;
	}
	inline long long& ctr(uint64_t t) { if(t != last_key || !last_ctr) { last_ctr = &taxo[t]; last_key = t; } return *last_ctr; }
	static inline long long num(const char* p, const char* e) { long long v = 0; bool neg = false; if(p < e && *p == '-') { neg = true; p++; } for(; p < e && *p >= '0' && *p <= '9'; p++) v = v * 10 + (*p - '0'); return neg ? -v : v; }
	std::vector<const char*> c;
	void consume(const char* p, size_t n) {                   // complete classification rows, header excluded
		const char* end = p + n;
		// the readID / taxID / score / hitLength fields wherever the column list puts them; rows with fewer fields
		// than the list are skipped
		const int want = (int)o.cols.fields.size() - 1;
		const int ci = o.kr_col[0], ct = o.kr_col[1], cs = o.kr_col[2], cl = o.kr_col[3];
		c.resize((size_t)want + 2);
		while(p < end) {
			const char* nl = (const char*)memchr(p, '\n', (size_t)(end - p));
			const char* le = nl ? nl : end;
			int k = 0; c[0] = p;
			for(const char* q = p; q < le && k < want; ) { const char* t = (const char*)memchr(q, '\t', (size_t)(le - q)); if(!t) break; c[++k] = t + 1; q = t + 1; }
			p = nl ? nl + 1 : end;
			if(k < want) continue;
			c[k + 1] = le + 1;                                        // field i ends at c[i + 1] - 1
			const char* id = c[ci]; const size_t idl = (size_t)(c[ci + 1] - 1 - c[ci]);
			if(o.kr_has_len && num(c[cl], c[cl + 1] - 1) < o.kr_min_len) continue;
			if(o.kr_has_score && num(c[cs], c[cs + 1] - 1) < o.kr_min_score) continue;
			uint64_t tax = 0; bool dotted = false;
			for(const char* q = c[ct]; q < c[ct + 1] - 1; q++) { if(*q == '.') { dotted = true; break; } tax = tax * 10 + (uint64_t)(*q - '0'); }
			if(dotted) { std::cerr << "Couldn't find parent of taxID " << std::string(c[ct], c[ct + 1] - 1) << " - directly assigned to root." << std::endl; tax = 1; }
			else if(!in_tree(tax)) tax = 1;
			if(have_prev && idl == prev_id.size() && memcmp(id, prev_id.data(), idl) == 0) {
				ctr(prev_tax) -= 1; prev_tax = lca(prev_tax, tax); ctr(prev_tax) += 1;
			} else { ctr(tax) += 1; seq_count++; prev_tax = tax; prev_id.assign(id, idl); }
			have_prev = true;
		}
	}
	static const char* rank_code(const char* r) {
		static const char* const tab[][2] = {{"species", "S"}, {"genus", "G"}, {"family", "F"}, {"order", "O"}, {"class", "C"}, {"phylum", "P"}, {"kingdom", "K"}, {"superkingdom", "D"}};
		for(size_t i = 0; i < 8; i++) if(strcmp(r, tab[i][0]) == 0) return tab[i][1];
		return "-";
	}
	void write() {
		if(seq_count <= 0) { std::cerr << "No sequence matches with given settings" << std::endl; return; }
		FILE* f = fopen(o.kreport.c_str(), "wb");
		if(!f) { std::cerr << "Error: could not open kreport file " << o.kreport << std::endl; return; }
		std::map<uint64_t, std::vector<uint64_t> > child;
		for(size_t i = 0; i < h.nodes.size(); i++) { const uint64_t t = h.nodes[i].taxid; child[t == 1 ? 0 : h.nodes[i].parent].push_back(t); }
		std::unordered_map<uint64_t, long long> clade(taxo.begin(), taxo.end());
		{   // dfs_summation(1), post-order
			std::vector<std::pair<uint64_t, size_t> > st; std::set<uint64_t> seen;
			st.push_back(std::make_pair((uint64_t)1, (size_t)0)); seen.insert(1);
			while(!st.empty()) {
				const uint64_t node = st.back().first; std::map<uint64_t, std::vector<uint64_t> >::const_iterator ch = child.find(node);
				if(ch != child.end() && st.back().second < ch->second.size()) {
					const uint64_t c = ch->second[st.back().second++];
					if(seen.insert(c).second) st.push_back(std::make_pair(c, (size_t)0));
				} else {
					st.pop_back();
					if(!st.empty()) { std::unordered_map<uint64_t, long long>::const_iterator v = clade.find(node); clade[st.back().first] += (v == clade.end() ? 0 : v->second); }
				}
			}
		}
		const double total = (double)seq_count;
		fprintf(f, "%6.2f\t%lld\t%lld\t%s\t%d\t%s%s\n", (double)clade[0] * 100 / total, clade[0], taxo[0], "U", 0, "", "unclassified");
		struct Frame { uint64_t node; int depth; };
		std::vector<Frame> st; st.push_back(Frame{1, 0});
		std::set<uint64_t> seen;
		while(!st.empty()) {
			const Frame fr = st.back(); st.pop_back();
			std::unordered_map<uint64_t, long long>::const_iterator cv = clade.find(fr.node);
			const long long cl = cv == clade.end() ? 0 : cv->second;
			if(!cl && !o.kr_zeros) continue;
			if(!seen.insert(fr.node).second) continue;
			std::unordered_map<uint64_t, long long>::const_iterator tv = taxo.find(fr.node);
			const TaxNode* nd = h.find_node(fr.node);
			std::map<uint64_t, std::string>::const_iterator nm = (fr.node >> 32) ? h.names.end() : h.names.find(fr.node);
			fprintf(f, "%6.2f\t%lld\t%lld\t%s\t%llu\t", (double)cl * 100 / total, cl, tv == taxo.end() ? 0ll : tv->second, rank_code(nd ? rank_name(nd->rank) : ""), (unsigned long long)fr.node);
			for(int i = 0; i < fr.depth; i++) fputs("  ", f);
			fputs(nm != h.names.end() ? nm->second.c_str() : "", f); fputc('\n', f);
			std::map<uint64_t, std::vector<uint64_t> >::const_iterator ch = child.find(fr.node);
			if(ch != child.end()) {
				std::vector<uint64_t> kids = ch->second;
				std::stable_sort(kids.begin(), kids.end(), [&](uint64_t a, uint64_t b) {
					std::unordered_map<uint64_t, long long>::const_iterator x = clade.find(a), y = clade.find(b);
					return (x == clade.end() ? 0 : x->second) > (y == clade.end() ? 0 : y->second); });
				for(size_t i = kids.size(); i-- > 0;) st.push_back(Frame{kids[i], fr.depth + 1});    // reversed: the stack pops them in sorted order
			}
		}
		fclose(f);
	}
};


// ------------------------------------------------------------------------------ text operator driver
// Well-formed FASTQ/FASTA goes to the device as raw bytes (cfb_text_submit): this thread only reads the
// file into pinned memory, counts line ends to cut spans at record boundaries, and writes the rows that
// come back.  Anything irregular is handed to the record-level reader below from the first byte of the
// span that failed, so the output never depends on the path taken.
__attribute__((target_clones("avx2", "default")))
static size_t count_nl(const unsigned char* p, size_t n) { size_t c = 0; for(size_t i = 0; i < n; i++) c += p[i] == '\n'; return c; }

struct SpanFile {        // one input file of a source, consumed in spans that end at record boundaries
	int fd = -1; uint64_t file_pos = 0, file_size = 0, span_start = 0; bool eof = false;
	std::vector<unsigned char> carry;              // bytes after the previous cut
	GzReader* gz = NULL;                           // gzip or bzip2 file: file_pos counts decompressed bytes
	bool open(const std::string& p) {
		// stat before open: opening and closing a FIFO (the `centrifuge` wrapper feeds compressed reads through mkfifo,
		// centrifuge:470-545) would leave its writer without a reader
		struct stat st; if(::stat(p.c_str(), &st) != 0 || !S_ISREG(st.st_mode)) return false;
		fd = ::open(p.c_str(), O_RDONLY);
		if(fd < 0) return false;
		if(fstat(fd, &st) != 0 || !S_ISREG(st.st_mode)) { ::close(fd); fd = -1; return false; }
		file_size = (uint64_t)st.st_size;
		posix_fadvise(fd, 0, 0, POSIX_FADV_SEQUENTIAL);
		if(const int fmt = compressed_format(fd)) {
			gz = new GzReader();
			const bool ok = gz->open(p, fd, fmt);
			fd = -1;
			if(!ok) return true;                       // reported by the first fill
		}
		return true;
	}
	void close() {
		if(gz) { gz->close(); delete gz; gz = NULL; }
		if(fd >= 0) ::close(fd);
		fd = -1;
	}
	const std::string& error() const { static const std::string none; return gz ? gz->err : none; }
	// fill buf (capacity cap) with carry + file bytes up to `want`; returns bytes in buf, line ends in *lines.
	// The file part is read by `threads` preads in parallel, each counting the line ends of its piece.
	size_t fill(unsigned char* buf, size_t cap, size_t want, size_t* lines, int threads) {
		size_t n = carry.size();
		if(n) memcpy(buf, carry.data(), n);
		span_start = file_pos - n;
		size_t nl = count_nl(buf, n);
		if(gz) {
			const size_t take = n < want ? std::min(want - n, cap - 1 - n) : 0;
			const size_t got = gz->err.empty() ? gz->read(buf + n, take) : 0;
			nl += count_nl(buf + n, got); n += got; file_pos += got;
			if(!gz->err.empty() || gz->peek() < 0) eof = true;
			if(eof && n > 0 && buf[n - 1] != '\n') { buf[n++] = '\n'; nl++; }
			*lines = nl;
			return n;
		}
		const uint64_t remain = file_size - file_pos;
		size_t take = n < want ? (size_t)std::min<uint64_t>(remain, std::min(want - n, cap - 1 - n)) : 0;
		if(take) {
			const int P = take >= (8u << 20) ? std::max(threads, 1) : 1;
			std::vector<size_t> got(P, 0), cnt(P, 0);
			auto piece = [&](int k) {
				const size_t lo = take * k / P, hi = take * (k + 1) / P; size_t done = lo, c = 0;
				while(done < hi) {      // 1 MB at a time so that the line-end count runs on cache-hot bytes
					const ssize_t r = pread(fd, buf + n + done, std::min<size_t>(hi - done, 1u << 20), (off_t)(file_pos + done));
					if(r <= 0) break;
					c += count_nl(buf + n + done, (size_t)r); done += (size_t)r;
				}
				got[k] = done - lo; cnt[k] = c;
			};
			std::vector<std::thread> th;
			for(int k = 1; k < P; k++) th.emplace_back(piece, k);
			piece(0);
			for(size_t k = 0; k < th.size(); k++) th[k].join();
			size_t ok = 0; bool shortfall = false;
			for(int k = 0; k < P; k++) { const size_t lo = take * k / P, hi = take * (k + 1) / P; if(shortfall) break; ok += got[k]; nl += cnt[k]; if(got[k] != hi - lo) shortfall = true; }
			if(shortfall) { nl = count_nl(buf, n + ok); }       // file shrank under us: keep the contiguous prefix
			n += ok; file_pos += ok;
			if(shortfall) file_size = file_pos;
		}
		if(file_pos >= file_size) eof = true;
		if(eof && n > 0 && buf[n - 1] != '\n') { buf[n++] = '\n'; nl++; }    // last line without a line end
		*lines = nl;
		return n;
	}
	// the byte that follows the last cut (first carried byte, else the next file byte); -1 at the end of the input
	int next_byte() {
		if(!carry.empty()) return carry[0];
		if(gz) return gz->peek();
		if(file_pos >= file_size) return -1;
		unsigned char c; return pread(fd, &c, 1, (off_t)file_pos) == 1 ? (int)c : -1;
	}
	// keep the first `keep_lines` lines of buf[0..n): returns the cut, stores the rest as carry
	size_t cut(const unsigned char* buf, size_t n, size_t lines, size_t keep_lines) {
		size_t end = n;
		for(size_t drop = lines - keep_lines + 1; drop > 0 && end > 0; drop--) {      // walk back over (lines - keep) line ends, land on the keep-th
			const void* q = memrchr(buf, '\n', end);
			if(!q) { end = 0; break; }
			end = (size_t)((const unsigned char*)q - buf);
		}
		const size_t c = keep_lines == 0 ? 0 : end + 1;
		carry.assign(buf + c, buf + n);
		return c;
	}
};

struct MultiKeyHash { size_t operator()(const std::string& k) const { uint64_t h = 1469598103934665603ull; for(size_t i = 0; i < k.size(); i++) { h ^= (unsigned char)k[i]; h *= 1099511628211ull; } return (size_t)h; } };
typedef std::unordered_map<std::string, uint64_t, MultiKeyHash> MultiObs;

struct TextStats { uint64_t spans = 0, units = 0, bytes_in = 0, bytes_out = 0, fallbacks = 0; double t_read = 0, t_gpu_wait = 0, t_write = 0, t_total = 0, t_submit = 0, t_setup = 0; };

template <class T> struct Chan {        // small blocking queue between the pipeline threads
	std::mutex mu; std::condition_variable cv; std::deque<T> q; bool closed = false;
	void push(const T& v) { { std::lock_guard<std::mutex> l(mu); q.push_back(v); } cv.notify_all(); }
	void close() { { std::lock_guard<std::mutex> l(mu); closed = true; } cv.notify_all(); }
	bool pop(T& v) { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return !q.empty() || closed; }); if(q.empty()) return false; v = q.front(); q.pop_front(); return true; }
};

// Three threads per source: a reader that fills pinned buffers and cuts spans at record boundaries, this
// thread submitting spans to the device(s) and collecting them in order, and a writer for the rows.  With several
// devices (--devices) span k goes to device k mod N: every device holds a replica of the index and its own context,
// spans are collected in submission order, so the output is the one-device output byte for byte.
struct TextPipe {
	std::vector<cfb_ctx*> ctxs; const Options& o; FILE* fo; MultiObs& multi; TextStats& st; KReport* kr = NULL;
	int S = 4; size_t cap = 0; int read_threads = 8;       // S spans per device: reader + 2 on the device + writer
	std::vector<unsigned char*> buf[2];
	TextPipe(const std::vector<cfb_ctx*>& c, const Options& o_, FILE* f, MultiObs& m, TextStats& s) : ctxs(c), o(o_), fo(f), multi(m), st(s) {
		const unsigned hw = std::thread::hardware_concurrency();
		if(hw) read_threads = (int)std::min<unsigned>(8, std::max<unsigned>(1, hw / 2));
		if(const char* e = getenv("CFB_READ_THREADS")) read_threads = std::max(1, atoi(e));
	}
	~TextPipe() { for(int m = 0; m < 2; m++) for(size_t i = 0; i < buf[m].size(); i++) cfb_host_free(buf[m][i]); }
	bool init(bool paired) {
		S = std::min(cfb_ctx_slots(ctxs[0]), 4); cap = 2 * o.text_block + 4096;
		const size_t want = (size_t)S * ctxs.size();
		for(int m = 0; m < (paired ? 2 : 1); m++) while(buf[m].size() < want) {
			unsigned char* p = (unsigned char*)cfb_host_alloc(cap);
			if(!p) return false;
			buf[m].push_back(p);
		}
		return true;
	}
	struct Span { int dev, slot; size_t bytes[2]; size_t rec; uint64_t start[2]; uint32_t hint; bool irregular; };
	struct Rows { int dev, slot; const char* tsv; uint64_t tsv_bytes; const uint64_t* multi; uint64_t n_multi; uint32_t stride; };

	// Runs one file (pair).  Returns 0 when it was consumed completely, 1 when the record-level reader has to
	// continue from byte offsets off[0..1] after `done` records, -1 on error.
	int run(const std::string& pa, const std::string* pb, uint64_t off[2], uint64_t& done) {
		const bool paired = pb != NULL; const size_t L = o.fasta ? 2 : 4; const int nm = paired ? 2 : 1;
		const int N = (int)ctxs.size();
		off[0] = off[1] = 0; done = 0;
		SpanFile f[2];
		if(!f[0].open(pa) || (paired && !f[1].open(*pb))) { f[0].close(); f[1].close(); return 1; }   // not a regular file: the stream reader handles it (and reports errors)
		const double t_setup0 = now_s();
		if(!init(paired)) { std::cerr << "Error: could not allocate pinned buffers" << std::endl; return -1; }
		const double t_begin = now_s();
		st.t_setup += t_begin - t_setup0;
		std::vector<Chan<int> > free_slots(N); Chan<Span> spans; Chan<Rows> rows;
		for(int d = 0; d < N; d++) for(int i = 0; i < S; i++) free_slots[d].push(i);
		std::atomic<bool> stop(false);
		double t_read = 0, t_write = 0;
		std::string read_err;

		std::thread reader([&] {
			bool first = true;
			for(uint64_t k = 0;; k++) {
				const int d = (int)(k % (uint64_t)N);
				int s;
				if(!free_slots[d].pop(s) || stop.load()) break;
				const int bi = d * S + s;
				const double t0 = now_s();
				Span sp; memset(&sp, 0, sizeof sp); sp.dev = d; sp.slot = s;
				size_t n[2] = {0, 0}, lines[2] = {0, 0};
				for(int m = 0; m < nm; m++) n[m] = f[m].fill(buf[m][bi], cap, o.text_block, &lines[m], read_threads);
				for(int m = 0; m < nm; m++) if(!f[m].error().empty() && read_err.empty()) read_err = f[m].error();
				if(!read_err.empty()) { t_read += now_s() - t0; break; }                        // compressed input failed: rows so far stand
				if(n[0] == 0 && (!paired || n[1] == 0)) { t_read += now_s() - t0; break; }      // input exhausted
				size_t rec = lines[0] / L;
				bool irregular = f[0].eof && lines[0] % L != 0;
				if(paired) { rec = std::min(rec, lines[1] / L); irregular |= f[1].eof && lines[1] % L != 0; }
				if(rec == 0) irregular = true;                       // a record longer than a span, or mates running out of step
				sp.start[0] = f[0].span_start; sp.start[1] = paired ? f[1].span_start : 0; sp.irregular = irregular; sp.rec = rec;
				if(!irregular) {
					for(int m = 0; m < nm; m++) sp.bytes[m] = f[m].cut(buf[m][bi], n[m], lines[m], rec * L);
					// A FASTA record runs up to the next '>' (pat.cpp:806-826), so its last line inside the span need not be
					// its end: unless the byte after the cut is '>' (or the input ends there), the tail record may continue in
					// the next span and is carried over whole; the wrapped record then sits inside one span, where the strict
					// layout check sees it and hands over to the record-level reader.
					if(o.fasta) {
						bool open_tail = false;
						for(int m = 0; m < nm; m++) { const int nb = f[m].next_byte(); if(nb >= 0 && nb != '>') open_tail = true; }
						if(open_tail) {
							rec -= 1; sp.rec = rec;
							if(rec == 0) { irregular = true; sp.irregular = true; }
							else for(int m = 0; m < nm; m++) sp.bytes[m] = f[m].cut(buf[m][bi], n[m], lines[m], rec * L);
						}
					}
				}
				if(!irregular) {
					if(first) {     // longest line in the head of the file sizes the first pass
						first = false; size_t longest = 0, ls = 0, line = 0; const size_t lim = std::min<size_t>(sp.bytes[0], 1u << 16);
						// integer quality lines are several bytes per base: they do not count
						const bool skip_quals = !o.fasta && o.quals.integer;
						for(size_t i = 0; i < lim; i++) if(buf[0][bi][i] == '\n') { if(!skip_quals || line % 4 != 3) longest = std::max(longest, i - ls); ls = i + 1; line++; }
						sp.hint = (uint32_t)std::min<size_t>(longest, 60000);
					}
				}
				t_read += now_s() - t0;
				spans.push(sp);
				if(irregular) break;
			}
			spans.close();
		});
		std::thread writer([&] {
			Rows r;
			while(rows.pop(r)) {
				const double t0 = now_s();
				if(r.tsv_bytes) fwrite(r.tsv, 1, r.tsv_bytes, fo);
				if(kr && r.tsv_bytes) kr->consume(r.tsv, r.tsv_bytes);
				for(uint64_t i = 0; i < r.n_multi; i++) {
					const uint64_t* rec = r.multi + i * r.stride;
					multi[std::string((const char*)(rec + 1), (size_t)rec[0] * 8)] += 1;
				}
				t_write += now_s() - t0;
				free_slots[r.dev].push(r.slot);
			}
		});

		cfb_text_opts to; memset(&to, 0, sizeof to);
		to.fasta = o.fasta ? 1 : 0; to.trim5 = o.trim5; to.trim3 = o.trim3; to.seed = o.seed;
		std::deque<Span> flight;          // submitted, oldest first
		int rc = 0; bool fallback = false; double t_wait = 0;
		auto collect_oldest = [&]() {
			const Span sp = flight.front(); flight.pop_front();
			cfb_text_result r;
			const double t0 = now_s();
			const int e = cfb_text_wait(ctxs[sp.dev], sp.slot, fallback ? 1 : 0, &r);
			t_wait += now_s() - t0;
			if(e != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; rc = -1; fallback = true; stop.store(true); free_slots[sp.dev].push(sp.slot); return; }
			if(fallback) { free_slots[sp.dev].push(sp.slot); return; }
			if(r.irregular) { fallback = true; stop.store(true); off[0] = sp.start[0]; off[1] = sp.start[1]; st.fallbacks++; free_slots[sp.dev].push(sp.slot); return; }
			done += r.n_units; st.spans++; st.units += r.n_units; st.bytes_out += r.tsv_bytes;
			Rows w; w.dev = sp.dev; w.slot = sp.slot; w.tsv = r.tsv; w.tsv_bytes = r.tsv_bytes; w.multi = r.multi; w.n_multi = r.n_multi; w.stride = r.multi_stride;
			rows.push(w);
		};
		for(;;) {
			Span sp;
			if(fallback || !spans.pop(sp)) break;
			if(sp.irregular) {
				while(!flight.empty() && !fallback) collect_oldest();
				if(!fallback) { fallback = true; off[0] = sp.start[0]; off[1] = sp.start[1]; st.fallbacks++; }
				free_slots[sp.dev].push(sp.slot);
				break;
			}
			if(sp.hint) to.maxlen_hint = sp.hint;
			const int bi = sp.dev * S + sp.slot;
			const double ts0 = now_s();
			if(cfb_text_submit(ctxs[sp.dev], sp.slot, buf[0][bi], sp.bytes[0], paired ? buf[1][bi] : NULL, sp.bytes[1], sp.rec, &to) != CFB_OK) {
				std::cerr << "Error: " << cfb_last_error() << std::endl; rc = -1; fallback = true; stop.store(true); free_slots[sp.dev].push(sp.slot); break;
			}
			st.t_submit += now_s() - ts0;
			st.bytes_in += sp.bytes[0] + sp.bytes[1];
			flight.push_back(sp);
			// keep every device two spans deep; collect the oldest as soon as one more is queued
			while((int)flight.size() > N * std::max(1, S - 2) && !fallback) collect_oldest();
		}
		while(!flight.empty()) collect_oldest();
		stop.store(true);
		for(int d = 0; d < N; d++) free_slots[d].close();
		{ Span sp; while(spans.pop(sp)) {} }      // reader may have queued spans after the failing one: they are re-read by the record reader
		reader.join();
		rows.close(); writer.join();
		f[0].close(); f[1].close();
		if(!read_err.empty()) { std::cerr << read_err << std::endl; rc = -1; }
		st.t_read += t_read; st.t_write += t_write; st.t_gpu_wait += t_wait; st.t_total += now_s() - t_begin;
		if(rc < 0) return -1;
		return fallback ? 1 : 0;
	}
};

// A list of read files behind one record counter, as BufferedFilePatternSource reads it (pat.h:786-811,883-904).
// centrifuge-class feeds it one file at a time (see cfb_run), which is also what decides its messages: a file that
// cannot be opened is the whole list, hence "No input read files were valid".
struct ListIn {
	std::vector<std::string> files; size_t next = 0; FileIn in; bool is_open = false, first = true;
	bool open_next() {                  // BufferedFilePatternSource::open
		while(next < files.size()) {
			const std::string& p = files[next++];
			if(in.open(p)) { is_open = true; first = true; return true; }
			std::cerr << "Warning: Could not open read file \"" << p << "\" for reading; skipping..." << std::endl;
		}
		std::cerr << "Error: No input read files were valid" << std::endl;
		throw 1;
	}
	// next record of the list; false when every file is exhausted
	bool read(bool fasta, Rec& r, uint64_t& count, int trim5, int trim3, bool keep_qual, const Quals& qe) {
		for(;;) {
			if(!is_open) { if(next >= files.size()) return false; open_next(); }
			const bool ok = fasta ? parse_fasta(in, r, count, first, trim5, trim3) : parse_fastq(in, r, count, first, trim5, trim3, keep_qual, qe);
			if(ok) return true;
			in.close(); is_open = false;
		}
	}
	void close() { if(is_open) in.close(); is_open = false; }
};

static void write_report(const HostIndex& h, const Options& o, Species& sp, int device, const std::string& path) {   // centrifuge.cpp:3231-3319
	std::cerr << "report file " << path << std::endl;
	std::ofstream ro(path.c_str());
	if(o.abundance) {
		size_t iters = 0; double diff = 0.0;
		calc_abundance(h, sp, iters, diff, device);
		std::cerr << "Number of iterations in EM algorithm: " << iters << std::endl;
		std::cerr << "Probability diff. (P - P_prev) in the last iteration: " << diff << std::endl;
	}
	ro << "name\ttaxID\ttaxRank\tgenomeSize\tnumReads\tnumUniqueReads\tabundance" << std::endl;
	for(std::map<uint64_t, Counts>::const_iterator it = sp.counts.begin(); it != sp.counts.end(); ++it) {
		const uint64_t taxid = it->first;
		if(taxid == 0) continue;
		std::map<uint64_t, std::string>::const_iterator nm = h.names.find(taxid);
		if(nm != h.names.end()) ro << nm->second; else ro << taxid;
		ro << '\t' << taxid << '\t';
		const TaxNode* n = h.find_node(taxid);
		const int rank = n ? n->rank : 0; const bool leaf = n ? n->leaf != 0 : false;
		if(rank == RANK_UNKNOWN && leaf) ro << "leaf"; else ro << rank_name(rank);
		ro << '\t';
		std::map<uint64_t, uint64_t>::const_iterator s = h.sizes.find(taxid);
		ro << (s != h.sizes.end() ? s->second : 0) << '\t' << it->second.n_reads << '\t' << it->second.n_unique << '\t';
		std::map<uint64_t, double>::const_iterator ab = sp.abundance_len.find(taxid);
		if(ab != sp.abundance_len.end()) ro << ab->second; else ro << "0.0";
		ro << std::endl;
	}
}

// --separator, after input `idx` (the -1/-2 pairs, then the -U files, from 0; centrifuge.cpp:3128-3223) once its rows
// are in `fo` and its counts in `sp`: the input's report goes to centrifuge_report_<idx>.tsv in the working directory,
// the per-taxon counts start again from zero, and "#File_End_Here" follows the rows.  The tie sets the EM runs over
// (`observed`) are kept, as the reference's metrics.reset() keeps them, so every later input's abundance column is
// computed over the tie sets of all inputs so far.  The report is closed before the separator line is flushed: the
// `centrifuge` wrapper renames the report once it has read that line, and only then feeds the next input into its FIFO.
static void end_input(const HostIndex& h, const Options& o, Species& sp, int device, size_t idx, FILE* fo) {
	write_report(h, o, sp, device, "centrifuge_report_" + std::to_string(idx) + ".tsv");
	sp.reset_counts();
	fputs("#File_End_Here\n", fo);
	fflush(fo);
}

static void print_arg_desc() {            // same shape as printArgDesc centrifuge.cpp:701-732
	for(const OptDesc* d = kLong; d->name; d++) std::cout << d->name << "\t" << d->has_arg << std::endl;
	const size_t n = strlen(kShort);
	for(size_t i = 0; i < n; i++) {
		if(i + 1 < n && kShort[i + 1] == ':') { std::cout << kShort[i] << "\t" << 1 << std::endl; i++; }
		else std::cout << kShort[i] << "\t" << 0 << std::endl;
	}
}

static int parse_args(int argc, const char** argv, Options& o, bool& exit_now) {
	cfb_params_default(&o.prm);
	exit_now = false;
	std::string rank_name_arg = "strain";
	int n_ceils = 0;
	for(int i = 1; i < argc; i++) {
		std::string a = argv[i];
		std::string key; bool is_long = false;
		if(a.size() > 2 && a[0] == '-' && a[1] == '-') { key = a.substr(2); is_long = true; }
		else if(a.size() >= 2 && a[0] == '-') key = a.substr(1, 1);
		else {   // positional: <index> then reads, as the reference's getopt tail does (centrifuge.cpp:1628-1660)
			if(o.index.empty()) o.index = a; else { std::vector<std::string> v = split(a, ','); o.singles.insert(o.singles.end(), v.begin(), v.end()); }
			continue;
		}
		std::string val; bool has_val = false;
		if(is_long) { size_t eq = key.find('='); if(eq != std::string::npos) { val = key.substr(eq + 1); key = key.substr(0, eq); has_val = true; } }
		else if(a.size() > 2) { val = a.substr(2); has_val = true; }
		int need = -1;
		if(is_long) { for(const OptDesc* d = kLong; d->name; d++) if(key == d->name) need = d->has_arg; }
		else { const char* q = strchr(kShort, key[0]); if(q && key[0] != ':') need = q[1] == ':' ? 1 : 0; }
		if(need < 0) { std::cerr << "centrifuge-class: unrecognized option '" << a << "'" << std::endl; return 1; }
		if(need == 1 && !has_val) { if(i + 1 >= argc) { std::cerr << "centrifuge-class: option '" << a << "' requires an argument" << std::endl; return 1; } val = argv[++i]; }
		if(key == "x") o.index = val;
		else if(key == "U") { std::vector<std::string> v = split(val, ','); o.singles.insert(o.singles.end(), v.begin(), v.end()); }
		else if(key == "1") { std::vector<std::string> v = split(val, ','); o.mates1.insert(o.mates1.end(), v.begin(), v.end()); }
		else if(key == "2") { std::vector<std::string> v = split(val, ','); o.mates2.insert(o.mates2.end(), v.begin(), v.end()); }
		else if(key == "f") o.fasta = true; else if(key == "q") o.fasta = false;
		else if(key == "S") o.out = val; else if(key == "report-file") o.report = val;
		else if(key == "k") { o.prm.khits = atoi(val.c_str()); if(o.prm.khits < 1) { std::cerr << "-k arg must be at least 1" << std::endl; return 1; } }
		else if(key == "min-hitlen") { o.prm.min_hitlen = atoi(val.c_str()); if(o.prm.min_hitlen < 15) { std::cerr << "--min-hitlen arg must be at least 15" << std::endl; return 1; } }
		else if(key == "host-taxids") { std::vector<std::string> v = split(val, ','); for(size_t k = 0; k < v.size(); k++) o.host.push_back(strtoull(v[k].c_str(), NULL, 10)); }
		else if(key == "exclude-taxids") { std::vector<std::string> v = split(val, ','); for(size_t k = 0; k < v.size(); k++) o.excl.push_back(strtoull(v[k].c_str(), NULL, 10)); }
		else if(key == "no-traverse") o.prm.tree_traverse = 0;
		else if(key == "classification-rank") rank_name_arg = val;
		else if(key == "no-abundance") o.abundance = false;
		else if(key == "p" || key == "threads" || key == "wrapper") { /* host threads are managed internally */ }
		else if(key == "reorder" || key == "mm") { /* output is always in input order; index is always resident in HBM */ }
		else if(key == "t" || key == "time") o.time = true;
		else if(key == "quiet") o.quiet = true;
		else if(key == "seed") o.seed = (uint32_t)strtoul(val.c_str(), NULL, 10);
		else if(key == "u" || key == "upto" || key == "qupto") o.upto = strtoull(val.c_str(), NULL, 10);
		else if(key == "s" || key == "skip") o.skip = strtoull(val.c_str(), NULL, 10);
		else if(key == "5" || key == "trim5") o.trim5 = atoi(val.c_str());
		else if(key == "3" || key == "trim3") o.trim3 = atoi(val.c_str());
		else if(key == "device") o.device = atoi(val.c_str());
		else if(key == "devices") {      // "0-7", "0,2,5", "all"
			o.devices.clear();
			if(val == "all") o.devices.push_back(-1);
			else {
				std::vector<std::string> parts = split(val, ',');
				for(size_t k = 0; k < parts.size(); k++) {
					const size_t dash = parts[k].find('-');
					const int lo = atoi(parts[k].substr(0, dash).c_str()), hi = dash == std::string::npos ? lo : atoi(parts[k].substr(dash + 1).c_str());
					if(lo < 0 || hi < lo || hi > 63) { std::cerr << "--devices arg must be a list of device numbers or ranges" << std::endl; return 1; }
					for(int d = lo; d <= hi; d++) if(std::find(o.devices.begin(), o.devices.end(), d) == o.devices.end()) o.devices.push_back(d);
				}
				if(o.devices.empty()) { std::cerr << "--devices arg must be a list of device numbers or ranges" << std::endl; return 1; }
			}
		}
		else if(key == "batch-units") o.batch_units = (size_t)strtoull(val.c_str(), NULL, 10);
		else if(key == "text-block-mb") { const size_t mb = (size_t)strtoull(val.c_str(), NULL, 10); o.text_block = std::min<size_t>(std::max<size_t>(mb, 1), 1024) << 20; }
		else if(key == "host-parse") o.host_parse = true;
		else if(key == "kreport-file") o.kreport = val;
		else if(key == "kreport-show-zeros") o.kr_zeros = true;
		else if(key == "kreport-min-score") { o.kr_has_score = true; o.kr_min_score = atoll(val.c_str()); }
		else if(key == "kreport-min-length") { o.kr_has_len = true; o.kr_min_len = atoll(val.c_str()); }
		else if(key == "tab-fmt-cols") { std::string err; if(!o.cols.parse(val, err)) { std::cerr << err << std::endl; return 1; } }   // the last one wins
		else if(key == "separator") o.separator = true;
		else if(key == "passthrough") { /* SAM XR:Z: tag only (centrifuge.cpp:1220-1223): no effect on tabular output */ }
		// Each --n-ceil is parsed as it is met.  The reference collects them all into its policy string first; when two are
		// malformed its first error line can name the other one (an empty token is checked for every setting before any
		// setting's type), which only matters for runs it refuses anyway.
		else if(key == "n-ceil") {
			if(n_ceils == 0) o.nceil = nceil_policy_init();
			std::string err; if(!nceil_parse(val, o.nceil, err, 5 + n_ceils++)) { std::cerr << err << std::endl; return 1; }
		}
		// --ignore-quals only changes mismatch penalties (centrifuge.cpp:1259,1548 -> Scoring); the classifier scores hits by
		// length and the per-read seed (genRandSeed pat.h:55-91) reads the qualities whatever it says
		else if(key == "ignore-quals") { }
		// --nofw / --norc only reach HI_Aligner::initRead (centrifuge.cpp:2594-2597, hi_aligner.h:739-772), which stores
		// them; Classifier::go (classifier.h) searches both strands regardless
		else if(key == "nofw" || key == "norc") { }
		// quality encodings, applied in command-line order (cf_quals.h)
		else if(o.quals.apply(key)) { }
		else if(key == "arg-desc") { print_arg_desc(); exit_now = true; return 0; }
		else if(key == "version") { std::cout << "centrifuge-class (cfb200, H100-native) compatible with Centrifuge 1.0.4" << std::endl; exit_now = true; return 0; }
		else if(key == "h" || key == "help") { std::cout << "Usage: centrifuge-class [options]* -x <cf-idx> {-1 <m1> -2 <m2> | -U <r>} [-S <out.tsv>] [--report-file <report>]" << std::endl; exit_now = true; return 0; }
	}
	o.prm.class_rank_slot = rank_to_slot(rank_from_name(rank_name_arg.c_str()));
	o.prm.host_taxids = o.host.data(); o.prm.n_host_taxids = o.host.size();
	o.prm.excluded_taxids = o.excl.data(); o.prm.n_excluded_taxids = o.excl.size();
	if(o.index.empty()) { std::cerr << "No index, query, or output file specified!" << std::endl; return 1; }
	if(o.mates1.size() != o.mates2.size()) { std::cerr << "Error: " << o.mates1.size() << " mate files/sequences were specified with -1, but " << o.mates2.size() << std::endl << "mate files/sequences were specified with -2.  The same number of mate files/" << std::endl << "sequences must be specified with -1 and -2." << std::endl; return 1; }
	if(o.singles.empty() && o.mates1.empty()) { std::cerr << "No index, query, or output file specified!" << std::endl; return 1; }
	if(o.batch_units < 1) o.batch_units = 1;
	if(o.separator && !o.kreport.empty()) { std::cerr << "Error: --kreport-file cannot be used with --separator (there is no per-input Kraken-style report)" << std::endl; return 1; }
	if(!o.kreport.empty()) {          // the Kraken-style report reads these fields of every row
		static const uint8_t need[4] = {COL_READ_ID, COL_TAX_ID, COL_SCORE, COL_HIT_LENGTH};
		for(int k = 0; k < 4; k++) {
			o.kr_col[k] = o.cols.index_of(need[k]);
			if(o.kr_col[k] < 0) { std::cerr << "Error: --kreport-file needs the readID, taxID, score and hitLength columns in --tab-fmt-cols" << std::endl; return 1; }
		}
	}
	// -s together with -u: rdids are shifted up by the skipped reads (centrifuge.cpp:1628-1633, 32-bit arithmetic)
	if(o.upto != std::numeric_limits<uint64_t>::max()) { const uint32_t u = (uint32_t)o.upto, sk = (uint32_t)o.skip; if((uint32_t)(u + sk) > u) o.upto = (uint32_t)(u + sk); }
	if(const char* e = getenv("CFB_TEXT_BLOCK")) o.text_block = std::max<size_t>((size_t)strtoull(e, NULL, 10), 4096);   // bytes; tests use tiny spans
	return 0;
}

}  // namespace

// Test hook (host only): run the record-level reader over a file and dump, per read, name / bases / seed / filter
// verdict, so that tests can diff it with the oracle's reader without a GPU.
extern "C" int cfb_test_parse_quals(const char* path, int fasta, int trim5, int trim3, uint32_t seed, const char* n_ceil, const char* quals, const char* out_path);
extern "C" int cfb_test_parse(const char* path, int fasta, int trim5, int trim3, uint32_t seed, const char* out_path) {
	return cfb_test_parse_quals(path, fasta, trim5, trim3, seed, NULL, NULL, out_path);
}
// the same under an --n-ceil function (NULL: the default); CFB_EINVAL when it does not parse
extern "C" int cfb_test_parse_nceil(const char* path, int fasta, int trim5, int trim3, uint32_t seed, const char* n_ceil, const char* out_path) {
	return cfb_test_parse_quals(path, fasta, trim5, trim3, seed, n_ceil, NULL, out_path);
}
// the same under a quality encoding: `quals` lists the options (names without dashes, comma-separated) in command-line
// order, and each row gets a fifth column, the read's qualities as readQual prints them, in hex.  NULL: phred33 and
// four columns.  CFB_EINVAL for a name that is not a quality-encoding option.
extern "C" int cfb_test_parse_quals(const char* path, int fasta, int trim5, int trim3, uint32_t seed, const char* n_ceil, const char* quals, const char* out_path) {
	if(!path || !out_path) return CFB_EINVAL;
	NCeil nc; std::string err;
	if(n_ceil) { nc = nceil_policy_init(); if(!nceil_parse(n_ceil, nc, err)) return CFB_EINVAL; }
	Quals qe;
	if(quals) for(const std::string& q : split(quals, ',')) if(!qe.apply(q)) return CFB_EINVAL;
	init_tables();
	FileIn in;
	if(!in.open(path)) return CFB_EIO;
	FILE* fo = fopen(out_path, "wb");
	if(!fo) { in.close(); return CFB_EIO; }
	int rc = CFB_OK;
	try {
		Rec r; uint64_t cnt = 0; bool first = true;
		for(;;) {
			const bool ok = fasta ? parse_fasta(in, r, cnt, first, trim5, trim3) : parse_fastq(in, r, cnt, first, trim5, trim3, quals != NULL, qe);
			if(!ok) break;
			fputs(r.name.c_str(), fo); fputc('\t', fo);
			for(size_t i = 0; i < r.seq.size(); i++) fputc("ACGTN"[r.seq[i]], fo);
			fprintf(fo, "\t%u\t%d", read_seed(r, seed), passes_filters(r.seq, nc) ? 1 : 0);
			if(quals) {
				fputc('\t', fo);
				if(fasta) for(size_t i = 0; i < r.seq.size(); i++) fputs("49", fo);          // 'I' (pat.cpp:828)
				else for(size_t i = 0; i < r.qual.size(); i++) fprintf(fo, "%02x", (unsigned)(uint8_t)r.qual[i]);
			}
			fputc('\n', fo);
		}
	} catch(int) { rc = 1; }
	fclose(fo); in.close();
	return rc;
}

// reads_a / reads_b are comma-separated file lists, read as cfb_run's record-level reader reads them
static void read_units(const Options& o, const char* reads_a, const char* reads_b, HostBatch& hb) {
	ListIn la, lb; const bool paired = reads_b != NULL;
	la.files = split(reads_a, ','); if(paired) lb.files = split(reads_b, ',');
	hb.clear(paired); hb.qual_mode = o.keep_qual() ? (o.fasta ? 2 : 1) : 0;
	uint64_t cntA = 0, cntB = 0; Rec ra, rb;
	for(;;) {
		const bool okA = la.read(o.fasta, ra, cntA, o.trim5, o.trim3, o.keep_qual(), o.quals);
		bool okB = true;
		if(paired) okB = lb.read(o.fasta, rb, cntB, o.trim5, o.trim3, o.keep_qual(), o.quals);
		if(!okA && paired && okB) { std::cerr << "Error, fewer reads in file specified with -1 than in file specified with -2" << std::endl; throw 1; }
		if(!okA) break;
		if(!okB) { std::cerr << "Error, fewer reads in file specified with -2 than in file specified with -1" << std::endl; throw 1; }
		hb.add(ra, paired ? &rb : NULL, o.seed, o.nceil);
	}
	la.close(); lb.close();
}

// Test hook (host only): everything cfb_run does around the device call on its record-level path -- reader, batch
// assembly, seeds and filters, tie selection, TSV rows, per-taxon metrics, EM, report, Kraken-style report -- with the
// classification records supplied by the caller (tests pass the oracle's), so the whole host side is checked
// against the reference without a GPU.  rec_off/recs follow cfb_result; units are reads or pairs in file order.
// cols: a --tab-fmt-cols list (NULL = the default columns); an unknown name returns CFB_EINVAL with the reference's
// message in cfb_last_error-style storage readable through cfb_test_cols_error.
static std::string g_test_cols_err;
extern "C" const char* cfb_test_cols_error(void) { return g_test_cols_err.c_str(); }
extern "C" int cfb_test_host_path_nceil(const char* index_base, const char* reads_a, const char* reads_b, int fasta, int khits, uint32_t seed,
                                        int trim5, int trim3, const uint32_t* rec_off, const cfb_rec* recs, uint64_t n_units,
                                        const char* cols, const char* n_ceil, const char* out_tsv, const char* out_report, const char* out_kreport);
extern "C" int cfb_test_host_path_cols(const char* index_base, const char* reads_a, const char* reads_b, int fasta, int khits, uint32_t seed,
                                       int trim5, int trim3, const uint32_t* rec_off, const cfb_rec* recs, uint64_t n_units,
                                       const char* cols, const char* out_tsv, const char* out_report, const char* out_kreport) {
	return cfb_test_host_path_nceil(index_base, reads_a, reads_b, fasta, khits, seed, trim5, trim3, rec_off, recs, n_units, cols, NULL,
	                                out_tsv, out_report, out_kreport);
}
// the same with the reader's filter flags under an --n-ceil value (NULL: the default); the records are the caller's
extern "C" int cfb_test_host_path_nceil(const char* index_base, const char* reads_a, const char* reads_b, int fasta, int khits, uint32_t seed,
                                        int trim5, int trim3, const uint32_t* rec_off, const cfb_rec* recs, uint64_t n_units,
                                        const char* cols, const char* n_ceil, const char* out_tsv, const char* out_report, const char* out_kreport) {
	if(!index_base || !reads_a || !rec_off || !out_tsv || !out_report) return CFB_EINVAL;
	init_tables();
	Options o; cfb_params_default(&o.prm);
	if(n_ceil) { std::string err; o.nceil = nceil_policy_init(); if(!nceil_parse(n_ceil, o.nceil, err)) return CFB_EINVAL; }
	if(cols && !o.cols.parse(cols, g_test_cols_err)) return CFB_EINVAL;
	if(out_kreport) {
		const uint8_t need[4] = {COL_READ_ID, COL_TAX_ID, COL_SCORE, COL_HIT_LENGTH};
		for(int k = 0; k < 4; k++) if((o.kr_col[k] = o.cols.index_of(need[k])) < 0) return CFB_EINVAL;
	}
	cfb_index* ix = NULL;
	if(cfb_index_load(index_base, -1, &ix) != CFB_OK) return CFB_EIO;
	int rc = CFB_OK;
	try {
		o.prm.khits = khits; o.fasta = fasta != 0; o.seed = seed; o.trim5 = trim5; o.trim3 = trim3; o.report = out_report;
		if(out_kreport) o.kreport = out_kreport;
		const HostIndex& h = *cfb_index_host(ix);
		HostBatch hb;
		read_units(o, reads_a, reads_b, hb);
		if(hb.n != n_units) throw 3;
		cfb_result res; res.n_units = n_units; res.n_recs = rec_off[n_units]; res.rec_off = rec_off; res.recs = recs;
		Species sp; Formatter fmt(h, o, sp); KReport kr(h, o);
		fmt.format_batch(hb, res);
		FILE* fo = fopen(out_tsv, "wb");
		if(!fo) throw 2;
		fputs(o.cols.header().c_str(), fo);
		if(!fmt.out.empty()) fwrite(fmt.out.data(), 1, fmt.out.size(), fo);
		fclose(fo);
		if(kr.enabled() && !fmt.out.empty()) kr.consume(fmt.out.data(), fmt.out.size());
		write_report(h, o, sp, -1, o.report);
		if(kr.enabled()) kr.write();
	} catch(int e) { rc = e; }
	cfb_index_free(ix);
	return rc;
}

// Test hook (host only): cfb_run's record-level path under --separator over n_inputs inputs, with the classification
// records supplied by the caller.  Input i is reads_a[i], paired with reads_b[i] when reads_b and reads_b[i] are set,
// and holds n_units[i] units; rec_off / recs follow cfb_result over the units of all inputs in order.  The TSV with its
// separator lines goes to out_tsv, the per-input reports to centrifuge_report_<i>.tsv in the working directory.
extern "C" int cfb_test_separator(const char* index_base, int n_inputs, const char* const* reads_a, const char* const* reads_b, int fasta,
                                  int khits, int abundance, const uint64_t* n_units, const uint32_t* rec_off, const cfb_rec* recs,
                                  const char* out_tsv) {
	if(!index_base || n_inputs < 0 || !reads_a || !n_units || !rec_off || !out_tsv) return CFB_EINVAL;
	init_tables();
	Options o; cfb_params_default(&o.prm);
	o.prm.khits = khits; o.fasta = fasta != 0; o.abundance = abundance != 0; o.separator = true;
	cfb_index* ix = NULL;
	if(cfb_index_load(index_base, -1, &ix) != CFB_OK) return CFB_EIO;
	FILE* fo = fopen(out_tsv, "wb");
	int rc = fo ? CFB_OK : CFB_EIO;
	try {
		const HostIndex& h = *cfb_index_host(ix);
		Species sp; Formatter fmt(h, o, sp);
		if(fo) fputs(o.cols.header().c_str(), fo);
		uint64_t u0 = 0;
		for(int i = 0; i < n_inputs && fo; i++) {
			HostBatch hb;
			read_units(o, reads_a[i], reads_b && reads_b[i] ? reads_b[i] : NULL, hb);
			if(hb.n != n_units[i]) throw 3;
			cfb_result res; res.n_units = hb.n; res.n_recs = rec_off[u0 + hb.n] - rec_off[u0]; res.rec_off = rec_off + u0; res.recs = recs;
			fmt.format_batch(hb, res);
			if(!fmt.out.empty()) fwrite(fmt.out.data(), 1, fmt.out.size(), fo);
			end_input(h, o, sp, -1, (size_t)i, fo);
			u0 += hb.n;
		}
	} catch(int e) { rc = e; }
	if(fo) fclose(fo);
	cfb_index_free(ix);
	return rc;
}
extern "C" int cfb_test_host_path(const char* index_base, const char* reads_a, const char* reads_b, int fasta, int khits, uint32_t seed,
                                  int trim5, int trim3, const uint32_t* rec_off, const cfb_rec* recs, uint64_t n_units,
                                  const char* out_tsv, const char* out_report, const char* out_kreport) {
	return cfb_test_host_path_cols(index_base, reads_a, reads_b, fasta, khits, seed, trim5, trim3, rec_off, recs, n_units, NULL, out_tsv, out_report, out_kreport);
}

// The host iteration on caller-provided flattened tables (what cfb_run uses for small tables); same contract as
// cfb_em_abundance, no device involved.
extern "C" int cfb_em_abundance_host(uint64_t n, uint64_t K, const uint64_t* count, const uint64_t* key_off, const uint32_t* target,
                                     const uint64_t* len, double* p, uint64_t* iters, double* last_diff) {
	if(!count || !key_off || !target || !len || !p || !iters || !last_diff || n == 0) return CFB_EINVAL;
	EmFlat f; f.count.assign(count, count + K); f.key_off.assign(key_off, key_off + K + 1); f.target.assign(target, target + key_off[K]); f.len.assign(len, len + n);
	for(uint64_t t = 0; t < key_off[K]; t++) if(target[t] >= n) return CFB_EINVAL;
	std::vector<double> pv(p, p + n); size_t it = 0; double diff = 0.0;
	em_iterate(f, pv, it, diff);
	std::copy(pv.begin(), pv.end(), p);
	*iters = it; *last_diff = diff;
	return CFB_OK;
}

// Stand-alone form of the same report: classification TSV file in, Kraken-style report out (host only).
extern "C" int cfb_kreport(const char* index_base, const char* tsv_path, const char* out_path, int show_zeros,
                           int has_min_score, long long min_score, int has_min_length, long long min_length) {
	if(!index_base || !tsv_path || !out_path) return CFB_EINVAL;
	cfb_index* ix = NULL;
	if(cfb_index_load(index_base, -1, &ix) != CFB_OK) return CFB_EIO;
	Options o; o.kreport = out_path; o.kr_zeros = show_zeros != 0; o.kr_has_score = has_min_score != 0; o.kr_min_score = min_score;
	o.kr_has_len = has_min_length != 0; o.kr_min_len = min_length;
	int rc = CFB_OK;
	{
		KReport kr(*cfb_index_host(ix), o);
		FILE* f = strcmp(tsv_path, "-") == 0 ? stdin : fopen(tsv_path, "rb");
		if(!f) rc = CFB_EIO;
		else {
			std::vector<char> buf(1 << 22); size_t have = 0; bool header = true;
			for(;;) {
				const size_t r = fread(buf.data() + have, 1, buf.size() - have, f);
				have += r;
				if(have == 0) break;
				size_t upto = have;
				if(r != 0) { const void* q = memrchr(buf.data(), '\n', have); upto = q ? (size_t)((const char*)q - buf.data()) + 1 : 0; }
				if(upto == 0 && r != 0) { buf.resize(buf.size() * 2); continue; }
				size_t from = 0;
				if(header) { const void* q = memchr(buf.data(), '\n', upto); from = q ? (size_t)((const char*)q - buf.data()) + 1 : upto; header = false; }
				kr.consume(buf.data() + from, upto - from);
				memmove(buf.data(), buf.data() + upto, have - upto); have -= upto;
				if(r == 0) break;
			}
			if(f != stdin) fclose(f);
			kr.write();
		}
	}
	cfb_index_free(ix);
	return rc;
}

// ------------------------------------------------------------------------------ centrifuge-promote
// In-process equivalent of the reference's `centrifuge-promote` script (SURVEY.md 8f rank 4): promote the taxIDs of a
// classification TSV to a rank ("genus", "family", ...) or, with level "lca", merge every read's rows into their lowest
// common ancestor.  Same bytes as the Perl script on the same TSV and index: rows of one read = consecutive rows with
// the same first column (centrifuge-promote:156-172), fields re-split on runs of tabs (:106,149), string-keyed
// taxonomy hashes fed by `centrifuge-inspect --taxonomy-tree` (:24-31), Perl's numeric / string comparison rules.
namespace {
struct Promote {
	std::unordered_map<std::string, std::string> parent, level;   // keyed by the taxid as centrifuge-inspect prints it
	std::string want;
	static double num(const std::string& s) {                       // Perl numification: leading number, else 0
		const char* p = s.c_str(); char* e = NULL;
		while(*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r' || *p == '\f' || *p == '\v') p++;
		const double v = strtod(p, &e);
		if(e == p) return 0.0;
		if(v != v) return 0.0;
		return v;
	}
	static std::vector<std::string> split_plus(const std::string& s) {      // split /\t+/: runs of tabs separate, trailing empty fields go
		std::vector<std::string> v; size_t i = 0; const size_t n = s.size();
		if(n == 0) return v;
		for(;;) {
			size_t j = s.find('\t', i);
			if(j == std::string::npos) { v.push_back(s.substr(i)); break; }
			v.push_back(s.substr(i, j - i));
			while(j < n && s[j] == '\t') j++;
			if(j >= n) break;
			i = j;
		}
		while(!v.empty() && v.back().empty()) v.pop_back();
		return v;
	}
	static std::string first_col(const std::string& s) { const size_t j = s.find('\t'); return j == std::string::npos ? s : s.substr(0, j); }   // split /\t/ -> [0]
	static std::string join(const std::vector<std::string>& c) { std::string o; for(size_t i = 0; i < c.size(); i++) { if(i) o.push_back('\t'); o += c[i]; } return o; }
	// PromoteTaxId (:43-58); `def` tells whether the argument was a defined value (an undefined parent numifies to 0)
	std::string promote(const std::string& tid, bool def) const {
		if(!def || num(tid) <= 0) return "0";
		std::unordered_map<std::string, std::string>::const_iterator lv = level.find(tid);
		if(lv == level.end()) return "0";
		if(lv->second == want) return tid;
		if(num(tid) <= 1) return "0";
		std::unordered_map<std::string, std::string>::const_iterator pa = parent.find(tid);
		if(pa == parent.end()) return promote("", false);
		return promote(pa->second, true);
	}
	std::string lca(std::string a, std::string b) const {            // :60-88 (`ge` is a STRING comparison, `>` a numeric one)
		if(a == "0") return b;
		if(b == "0") return a;
		if(a == b) return a;
		std::set<std::string> path;
		while(a.compare("1") >= 0) {
			path.insert(a);
			std::unordered_map<std::string, std::string>::const_iterator pa = parent.find(a);
			if(pa == parent.end()) { std::cerr << "Couldn't find parent of taxID " << a << " - directly assigned to root." << std::endl; break; }
			if(a == pa->second) break;
			a = pa->second;
		}
		while(num(b) > 1) {
			if(path.count(b)) return b;
			std::unordered_map<std::string, std::string>::const_iterator pb = parent.find(b);
			if(pb == parent.end()) { std::cerr << "Couldn't find parent of taxID " << b << " - directly assigned to root." << std::endl; break; }
			if(b == pb->second) break;
			b = pb->second;
		}
		return "1";
	}
	void flush(const std::vector<std::string>& lines, FILE* fo) const {      // OutputPromotedLines :90-153
		if(lines.empty()) return;
		std::vector<std::string> out; unsigned long long matches = 0;
		if(want != "lca") {
			std::set<std::string> seen;
			for(size_t i = 0; i < lines.size(); i++) {
				std::vector<std::string> c = split_plus(lines[i]);
				const bool has2 = c.size() > 2;
				std::string nt = promote(has2 ? c[2] : std::string(), has2);
				if(num(nt) <= 1) nt = has2 ? c[2] : std::string();
				std::string nl = c.size() > 1 ? c[1] : std::string();
				if(num(nt) >= 1) { std::unordered_map<std::string, std::string>::const_iterator lv = level.find(nt); if(lv != level.end()) nl = lv->second; }
				if(!seen.insert(nt).second) continue;
				matches++;
				if(c.size() < 3) c.resize(3);
				c[2] = nt; c[1] = nl;
				out.push_back(join(c));
			}
		} else {
			matches = 1;
			std::vector<std::string> c = split_plus(lines[0]);
			std::string l = c.size() > 2 ? c[2] : std::string();
			for(size_t i = 1; i < lines.size(); i++) { std::vector<std::string> d = split_plus(lines[i]); l = lca(l, d.size() > 2 ? d[2] : std::string()); }
			if(c.size() < 3) c.resize(3);
			if(l != c[2]) { std::unordered_map<std::string, std::string>::const_iterator lv = level.find(l); c[1] = lv != level.end() ? lv->second : std::string(); }
			c[2] = l;
			out.push_back(join(c));
		}
		char nb[32]; snprintf(nb, sizeof nb, "%llu", matches);
		for(size_t i = 0; i < out.size(); i++) {
			std::vector<std::string> c = split_plus(out[i]);
			if(c.empty()) c.push_back(nb); else c.back() = nb;
			const std::string row = join(c);
			fwrite(row.data(), 1, row.size(), fo); fputc('\n', fo);
		}
	}
};
}  // namespace

// centrifuge-promote <index> <classification TSV> <level> > out   (out_path "-" = stdout).  Host only.
extern "C" int cfb_promote(const char* index_base, const char* tsv_path, const char* level, const char* out_path) {
	if(!index_base || !tsv_path || !level || !out_path) return CFB_EINVAL;
	cfb_index* ix = NULL;
	if(cfb_index_load(index_base, -1, &ix) != CFB_OK) return CFB_EIO;
	int rc = CFB_OK;
	{
		const HostIndex& h = *cfb_index_host(ix);
		Promote pr; pr.want = level;
		for(size_t i = 0; i < h.nodes.size(); i++) {
			char a[32], b[32]; snprintf(a, sizeof a, "%llu", (unsigned long long)h.nodes[i].taxid); snprintf(b, sizeof b, "%llu", (unsigned long long)h.nodes[i].parent);
			pr.parent[a] = b; pr.level[a] = rank_name(h.nodes[i].rank);
		}
		std::ifstream in; std::istream* is = &std::cin;
		if(strcmp(tsv_path, "-") != 0) { in.open(tsv_path, std::ios::binary); if(!in) rc = CFB_EIO; is = &in; }
		FILE* fo = rc == CFB_OK ? (strcmp(out_path, "-") == 0 ? stdout : fopen(out_path, "wb")) : NULL;
		if(rc == CFB_OK && !fo) rc = CFB_EIO;
		if(rc == CFB_OK) {
			std::string line;
			if(std::getline(*is, line)) { fwrite(line.data(), 1, line.size(), fo); if(!is->eof()) fputc('\n', fo); }      // header, as read
			std::string prev; std::vector<std::string> lines;
			while(std::getline(*is, line)) {
				const std::string id = Promote::first_col(line);
				if(id == prev) lines.push_back(line);
				else { prev = id; pr.flush(lines, fo); lines.clear(); lines.push_back(line); }
			}
			pr.flush(lines, fo);
			if(fo != stdout) fclose(fo); else fflush(stdout);
		}
	}
	cfb_index_free(ix);
	return rc;
}

// everything a run owns, released on every way out (normal return, reader error -> throw 1, exception)
struct RunState {
	std::vector<cfb_index*> ix; std::vector<cfb_ctx*> ctx; FILE* fo = NULL;
	~RunState() {
		if(fo && fo != stdout) fclose(fo); else if(fo) fflush(stdout);
		for(size_t i = 0; i < ctx.size(); i++) if(ctx[i]) cfb_ctx_destroy(ctx[i]);      // waits for batches still in flight
		for(size_t i = 0; i < ix.size(); i++) if(ix[i]) cfb_index_free(ix[i]);
	}
};

extern "C" int cfb_run(int argc, const char** argv) {
	init_tables();
	Options o; bool exit_now = false;
	try {
		int rc = parse_args(argc, argv, o, exit_now);
		if(rc || exit_now) return rc;
		const auto t_start = std::chrono::steady_clock::now();
		RunState rs;
		// ---- devices: one replica of the index and one context per GPU
		std::vector<int> devs = o.devices;
		if(devs.size() == 1 && devs[0] == -1) { devs.clear(); int n = cfb_device_count(); for(int d = 0; d < n; d++) devs.push_back(d); if(devs.empty()) { std::cerr << "Error: no CUDA device (this build has no CPU fallback)" << std::endl; return 1; } }
		if(devs.empty()) devs.push_back(o.device);
		const int N = (int)devs.size();
		g_gz_device = devs[0];
		// File-to-file runs are bounded by the file system (tens of M reads/s), far below what the plain kernels
		// deliver (~180 M reads/s), so the tables that buy the last factor of two on the device (resolve table, walk8:
		// ~0.75 s per Gbp to build) would only delay the first read.  CFB_FULL_TABLES=1 builds them anyway.
		const uint32_t load_flags = getenv("CFB_FULL_TABLES") ? 0u : (CFB_LOAD_NO_RESOLVE_TABLE | CFB_LOAD_NO_WALK8);
		rs.ix.assign(N, (cfb_index*)NULL); rs.ctx.assign(N, (cfb_ctx*)NULL);
		{
			std::vector<std::string> errs(N); std::vector<std::thread> th;
			auto load_one = [&](int i) {
				if(cfb_index_load_ex(o.index.c_str(), devs[i], load_flags, &rs.ix[i]) != CFB_OK) { errs[i] = cfb_last_error(); return; }
				if(cfb_ctx_create(rs.ix[i], &o.prm, &rs.ctx[i]) != CFB_OK) { errs[i] = cfb_last_error(); return; }
				if(!o.nceil.is_default() && cfb_ctx_set_n_ceil(rs.ctx[i], o.nceil.type, o.nceil.c, o.nceil.l, o.nceil.mn, o.nceil.mx) != CFB_OK) { errs[i] = cfb_last_error(); return; }
				if(!o.quals.is_default() && cfb_ctx_set_quals(rs.ctx[i], o.quals.solexa, o.quals.phred64, o.quals.integer) != CFB_OK) errs[i] = cfb_last_error();
			};
			for(int i = 1; i < N; i++) th.emplace_back(load_one, i);
			load_one(0);
			for(size_t i = 0; i < th.size(); i++) th[i].join();
			for(int i = 0; i < N; i++) if(!errs[i].empty()) { std::cerr << "Error: " << errs[i] << std::endl; return 1; }
		}
		if(N > 1 && cfb_comm_init_all(rs.ctx.data(), N) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return 1; }
		cfb_ctx* ctx = rs.ctx[0];               // the record-level reader works on the first device
		const HostIndex& h = *cfb_index_host(rs.ix[0]);
		const auto t_loaded = std::chrono::steady_clock::now();
		FILE* fo = rs.fo = o.out == "-" ? stdout : fopen(o.out.c_str(), "wb");
		if(!fo) { std::cerr << "Error: could not open output file " << o.out << std::endl; return 1; }
		fputs(o.cols.header().c_str(), fo);
		Species sp; Formatter fmt(h, o, sp); KReport kr(h, o);
		const int nslots = std::min(cfb_ctx_slots(ctx), 4);
		std::vector<HostBatch> hb(nslots);
		for(int s = 0; s < nslots; s++) hb[s].qual_mode = o.keep_qual() ? (o.fasta ? 2 : 1) : 0;
		std::vector<bool> busy(nslots, false);
		int cur = 0;
		bool failed = false;
		auto drain = [&](int s) -> bool {
			cfb_result res;
			if(cfb_classify_wait(ctx, s, &res) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			fmt.format_batch(hb[s], res);
			if(!fmt.out.empty()) fwrite(fmt.out.data(), 1, fmt.out.size(), fo);
			if(kr.enabled() && !fmt.out.empty()) kr.consume(fmt.out.data(), fmt.out.size());
			busy[s] = false;
			return true;
		};
		auto flush = [&](int s) -> bool {
			if(hb[s].n == 0) return true;
			cfb_batch b; memset(&b, 0, sizeof b);
			b.n_units = hb[s].n; b.n_mates = hb[s].paired ? 2 : 1; b.bases = hb[s].bases.data(); b.n_bases = hb[s].bases.size();
			b.off[0] = hb[s].off[0].data(); b.len[0] = hb[s].len[0].data();
			if(hb[s].paired) { b.off[1] = hb[s].off[1].data(); b.len[1] = hb[s].len[1].data(); }
			b.flags = hb[s].flags.data();
			if(cfb_classify_submit(ctx, s, &b) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			busy[s] = true;
			return true;
		};
		// Centrifuge handles its inputs one by one (centrifuge.cpp:3006-3046: "the name is not plural here"): every -1/-2
		// file pair, then every -U file, gets a pattern source of its own, so the record counter that names unnamed reads
		// and drives --skip/--upto restarts with every file and mate files must hold the same number of records pair by
		// pair.  (bowtie2's one-source-per-list wiring in pat.cpp:330-420 is fed single-file lists; checked against the
		// binary: unnamed reads of a second -U file are named 0, 1, ...)  The metrics run on across files (:3231).
		struct Src { std::vector<std::string> a, b; bool paired; };
		std::vector<Src> srcs;
		for(size_t i = 0; i < o.mates1.size(); i++) { Src s; s.a.push_back(o.mates1[i]); s.b.push_back(o.mates2[i]); s.paired = true; srcs.push_back(s); }
		for(size_t i = 0; i < o.singles.size(); i++) { Src s; s.a.push_back(o.singles[i]); s.paired = false; srcs.push_back(s); }
		bool stop = false;
		MultiObs multi; TextStats tstats; uint64_t host_units = 0;
		TextPipe pipe(rs.ctx, o, fo, multi, tstats);
		if(kr.enabled()) pipe.kr = &kr;
		// device-side counters and the text operator's tie sets -> the host maps, for the units the text operator
		// classified since the last fold
		uint64_t folded = 0;
		auto fold_counts = [&]() -> bool {
			if(tstats.units == folded) return true;
			folded = tstats.units;
			// several devices: one NCCL all-reduce (sum, u64) of the per-taxon counters over the replicas' contexts
			const int global = N > 1 ? 1 : 0;
			if(N > 1 && cfb_counts_allreduce(rs.ctx.data(), N, NULL, 0) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			uint64_t n = 0;
			if(cfb_counts_read(ctx, global, NULL, NULL, NULL, NULL, 0, &n) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			std::vector<uint64_t> tx(n), nr(n), nu(n), no(n);
			if(n && cfb_counts_read(ctx, global, tx.data(), nr.data(), nu.data(), no.data(), n, &n) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			for(uint64_t i = 0; i < n; i++) {
				Counts& c = sp.counts[tx[i]]; c.n_reads += nr[i]; c.n_unique += nu[i];
				if(no[i]) sp.observed[std::vector<uint64_t>(1, tx[i])] += no[i];
			}
			for(MultiObs::const_iterator it = multi.begin(); it != multi.end(); ++it) {      // sparse tie sets: merged on the host, as SpeciesMetrics::merge does
				std::vector<uint64_t> ids(it->first.size() / 8);
				memcpy(ids.data(), it->first.data(), ids.size() * 8);
				sp.observed[ids] += it->second;
			}
			return true;
		};
		// --separator: input si is complete, from the text operator, the record-level reader or both.  Its counters
		// leave the devices and its tie sets the text operator's map before its report is written.
		auto separate = [&](size_t si) -> bool {
			if(!fold_counts()) return false;
			for(int i = 0; i < N; i++) if(cfb_counts_reset(rs.ctx[i]) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return false; }
			multi.clear();
			end_input(h, o, sp, devs[0], si, fo);
			return true;
		};
		const bool text_ok = !o.host_parse && !getenv("CFB_HOST_PARSE") && o.prm.khits <= 32 && o.skip == 0 && o.upto == std::numeric_limits<uint64_t>::max()
		                     && o.cols.fields.size() <= (size_t)kTextMaxCols;
		if(text_ok) for(int i = 0; i < N; i++) if(cfb_ctx_set_columns(rs.ctx[i], o.cols.spec().c_str()) != CFB_OK) { std::cerr << "Error: " << cfb_last_error() << std::endl; return 1; }
		for(size_t si = 0; si < srcs.size() && !failed && !stop; si++) {
			const Src& src = srcs[si];
			g_input_seq = si + 1;
			uint64_t off[2] = {0, 0}, cntA = 0, cntB = 0;      // cnt: records of this list read so far (PatternSource::readCnt_)
			size_t fi = 0;
			// whole files go through the text operator while they stay regular and the mate files stay in step
			while(text_ok && fi < src.a.size() && src.a[fi] != "-" && !(src.paired && src.b[fi] == "-")) {
				uint64_t done = 0;
				const int r = pipe.run(src.a[fi], src.paired ? &src.b[fi] : NULL, off, done);
				if(r < 0) { failed = true; break; }
				cntA += done; cntB += done;
				if(r != 0) break;                  // the record-level reader continues inside file fi, at off[]
				off[0] = off[1] = 0; fi++;
			}
			if(failed || fi >= src.a.size()) {
				if(!failed && o.separator && !separate(si)) failed = true;
				continue;
			}
			ListIn la, lb;
			la.files.assign(src.a.begin() + fi, src.a.end());
			if(src.paired) lb.files.assign(src.b.begin() + fi, src.b.end());
			// continue after the spans the text operator consumed: same parser state as if it had read them itself
			auto resume = [&](ListIn& l, uint64_t at) {
				if(at == 0) return;
				l.open_next(); l.in.seek(at); l.first = false;
				FileIn& f = l.in;
				if(!o.fasta) { while(f.peek() == '\n' || f.peek() == '\r') f.get(); f.get(); }   // the '@' that ends the previous record's parse
				else { while(f.peek() >= 0 && f.peek() != '>') f.get(); }   // the previous record's sequence loop runs up to the next '>' (blank lines at a span start belong to it)
			};
			resume(la, off[0]);
			if(src.paired) resume(lb, off[1]);
			Rec ra, rb;
			hb[cur].clear(src.paired);
			for(;;) {
				const uint64_t id = cntA;          // rdid of this read: the list's own record counter (pat.h:603-611)
				const bool okA = la.read(o.fasta, ra, cntA, o.trim5, o.trim3, o.keep_qual(), o.quals);
				bool okB = true;
				if(src.paired) okB = lb.read(o.fasta, rb, cntB, o.trim5, o.trim3, o.keep_qual(), o.quals);
				if(!okA && src.paired && okB) { std::cerr << "Error, fewer reads in file specified with -1 than in file specified with -2" << std::endl; throw 1; }
				if(!okA) break;
				if(!okB) { std::cerr << "Error, fewer reads in file specified with -2 than in file specified with -1" << std::endl; throw 1; }
				// empty reads are kept: the reference reports them as length-filtered "unclassified" rows
				// -s/-u count the records of each input, and the reference reads every input up to -u.  The run without
				// --separator ends at the first input that reaches -u instead (DESIGN.md 5).
				if(id >= o.upto) { stop = !o.separator; break; }
				if(id < o.skip) continue;
				hb[cur].add(ra, src.paired ? &rb : NULL, o.seed, o.nceil); host_units++;
				if(hb[cur].n >= o.batch_units) {
					if(!flush(cur)) { failed = true; break; }
					const int nxt = (cur + 1) % nslots;
					if(busy[nxt] && !drain(nxt)) { failed = true; break; }
					cur = nxt; hb[cur].clear(src.paired);
				}
			}
			la.close(); lb.close();
			if(failed) break;
			// finish this source: submit the partial batch, then drain everything in submission order
			if(!flush(cur)) { failed = true; break; }
			for(int k = 1; k <= nslots; k++) { const int s = (cur + k) % nslots; if(busy[s] && !drain(s)) { failed = true; break; } }
			hb[cur].clear(false);
			if(o.separator && !separate(si)) { failed = true; break; }
		}
		if(!failed && !o.separator && !fold_counts()) failed = true;
		if(getenv("CFB_TEXT_STATS")) {
			const auto t_done = std::chrono::steady_clock::now();
			cfb_index_tables tb; memset(&tb, 0, sizeof tb); cfb_index_get_tables(rs.ix[0], &tb);
			std::cerr << "[cfb] index load " << std::chrono::duration<double>(t_loaded - t_start).count() << " s (" << (tb.rank16_bytes ? "rank16" : "compact")
			          << " rank layout), reads " << std::chrono::duration<double>(t_done - t_loaded).count() << " s" << std::endl;
			std::cerr << "[cfb] text operator: " << tstats.units << " units in " << tstats.spans << " spans (" << tstats.bytes_in << " bytes in, " << tstats.bytes_out
			          << " bytes out, " << tstats.fallbacks << " fallbacks); record-level reader: " << host_units << " units" << std::endl;
			uint64_t lt[4] = {0, 0, 0, 0};
			for(cfb_ctx* x : rs.ctx) { uint64_t v[4]; if(cfb_ctx_long_stats(x, v) == CFB_OK) for(int i = 0; i < 4; i++) lt[i] += v[i]; }
			std::cerr << "[cfb] long units: " << lt[0] << " (" << lt[1] << " bases), " << lt[2] << " partial searches in segment chains, "
			          << lt[3] << " re-searched at the join" << std::endl;
			std::cerr << "[cfb] text pipeline " << tstats.t_total << " s: reader busy " << tstats.t_read << " s, device wait " << tstats.t_gpu_wait << " s, writer busy " << tstats.t_write << " s, submit " << tstats.t_submit << " s, pinned setup " << tstats.t_setup << " s" << std::endl;
			if(N > 1) std::cerr << "[cfb] " << N << " devices, per-taxon counters reduced with NCCL" << std::endl;
			if(g_gz.files) std::cerr << "[cfb] gunzip: " << g_gz.st[0] << " members, " << g_gz.st[1] << " bytes in, " << g_gz.st[2] << " bytes out, " << g_gz.st[3]
			                         << " chunks, " << g_gz.st[4] << " re-decoded, " << g_gz.t << " s" << std::endl;
			if(g_bz.files) std::cerr << "[cfb] bunzip2: " << g_bz.st[0] << " streams, " << g_bz.st[1] << " bytes in, " << g_bz.st[2] << " bytes out, " << g_bz.st[3]
			                         << " blocks, " << g_bz.st[4] << " rejected block starts, " << g_bz.t << " s" << std::endl;
		}
		if(fo != stdout) fclose(fo); else fflush(stdout);
		rs.fo = NULL;
		if(!failed && !o.report.empty() && !o.separator) write_report(h, o, sp, devs[0], o.report);   // --separator: every input had its own
		if(!failed && kr.enabled()) kr.write();
		return failed ? 1 : 0;
	} catch(int e) {
		return e ? e : 1;
	} catch(std::exception& e) {
		std::cerr << "Error: Encountered exception: '" << e.what() << "'" << std::endl;
		return 1;
	}
}
