// cf_build.cu -- GPU index builder: FASTA (or counter-based synthetic genomes) -> `.1-.4.cf`.
//
// Produces the files centrifuge-build-bin writes (byte-identical on the fixtures in tests/):
//   header / plen / rstarts / names      bt2_io.h:854-929,989-1030, bt2_idx.h:3235-3360,1630-1636
//   BWT sides + occ, zOff, fchr, ftab/eftab, SA sample of sequence ids, boundary rows
//                                        Ebwt::buildToDisk bt2_idx.h:3379-3840
//   .3.cf taxonomy tables                bt2_idx.h:1329-1506
// The reference sorts suffixes blockwise on the CPU (blockwise_sa.h); here the suffix array is
// never materialised as a whole: suffixes are bucketed by their first two bases, each bucket is
// radix-sorted on the GPU by successive 29-base windows of the 2-bit packed text (only groups that
// are still tied are refined), and every sorted bucket is immediately turned into BWT bases,
// sampled sequence ids, ftab counts and boundary rows, then dropped.
// Sorting primitives are CUB (library code; this is not the classification hot path).
#include "../../include/cfb200.h"
#include "cf_index.h"
#include "cf_synth.h"
#include "cf_buf.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <cctype>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <map>
#include <set>
#include <sstream>
#include <string>
#include <vector>

using namespace cfb;

namespace {

thread_local std::string g_berr;
int bfail(int code, const char* fmt, ...) {
	char b[512]; va_list ap; va_start(ap, fmt); vsnprintf(b, sizeof b, fmt, ap); va_end(ap); g_berr = b; return code;
}
#define BCK(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) return bfail(CFB_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while(0)

static const int kWin = 29;            // bases per refinement window (58 bits) + 6 bits of length code

// ---------------------------------------------------------------------------- device helpers
// text: base i in bits 62-2*(i&31) of word i>>5 (first base of a word most significant); zero padded
__device__ __forceinline__ uint64_t window32(const uint64_t* t, uint64_t i) {
	const uint64_t w = i >> 5; const unsigned s = (unsigned)(i & 31) * 2;
	const uint64_t a = t[w];
	if(s == 0) return a;
	return (a << s) | (t[w + 1] >> (64 - s));
}
__device__ __forceinline__ int base_at(const uint64_t* t, uint64_t i) { return (int)((t[i >> 5] >> (62 - 2 * (i & 31))) & 3); }

// The reference's suffix order treats the end of the text as GREATER than any base ("prefixes are
// lexicographically greater than their extensions", multikey_qsort.h:194-205,379).
// Sort key of suffix `pos` for the window starting d bases into the suffix: 29 bases, positions past
// the end padded with T (the largest base), and in the low bits a code that is 0 while the window is
// completely inside the text and grows as the suffix gets shorter -- so a suffix that ends inside the
// window sorts after every longer suffix with the same padded bases, shortest last.
__device__ __forceinline__ uint64_t suffix_key(const uint64_t* t, uint64_t len, uint64_t pos, uint64_t d) {
	const uint64_t R = len - pos;
	uint64_t chars = (1ull << 58) - 1;
	if(R > d) {
		chars = window32(t, pos + d) >> 6;
		const uint64_t r = R - d;
		if(r < (uint64_t)kWin) chars |= (1ull << (2 * (kWin - r))) - 1;
	}
	uint64_t real = 0;
	if(R + 2 >= d) { real = R + 2 - d; if(real > (uint64_t)kWin + 2) real = kWin + 2; }
	return (chars << 6) | ((uint64_t)kWin + 2 - real);
}
// 2-base bucket of suffix i; a suffix of length 1 is padded with T
__device__ __forceinline__ int bucket_of(const uint64_t* t, uint64_t len, uint64_t i) {
	int b = (int)(window32(t, i) >> 60);
	if(i + 1 >= len) b |= 3;
	return b;
}

struct InBucket {
	const uint64_t* t; uint64_t len; int b;
	__device__ __forceinline__ bool operator()(const uint64_t& i) const { return bucket_of(t, len, i) == b; }
};

__global__ void k_pack_text(const uint8_t* codes, uint64_t n, uint64_t* words, uint64_t nwords) {
	const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(w >= nwords) return;
	uint64_t v = 0;
	for(int k = 0; k < 32; k++) { const uint64_t i = w * 32 + k; if(i < n) v |= (uint64_t)(codes[i] & 3) << (62 - 2 * k); }
	words[w] = v;
}
__global__ void k_synth_text(SynthSpec sp, uint64_t* words, uint64_t nwords, uint64_t n) {
	const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(w >= nwords) return;
	uint64_t v = 0;
	for(int k = 0; k < 32; k++) {
		const uint64_t i = w * 32 + k;
		if(i < n) { const uint32_t seq = (uint32_t)(i / sp.len); v |= (uint64_t)synth_base(sp, seq, i - (uint64_t)seq * sp.len) << (62 - 2 * k); }
	}
	words[w] = v;
}
__global__ void k_bucket_hist(const uint64_t* t, uint64_t len, unsigned long long* hist) {
	__shared__ unsigned int sh[16];
	if(threadIdx.x < 16) sh[threadIdx.x] = 0;
	__syncthreads();
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) atomicAdd(&sh[bucket_of(t, len, i)], 1u);
	__syncthreads();
	if(threadIdx.x < 16) atomicAdd(&hist[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}
__global__ void k_keys(const uint64_t* t, uint64_t len, const uint64_t* pos, uint32_t n, uint64_t d, uint64_t* key) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if(j < n) key[j] = suffix_key(t, len, pos[j], d);
}
__global__ void k_heads(const uint64_t* key, uint32_t n, uint8_t* head) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if(j < n) head[j] = (j == 0 || key[j] != key[j - 1]) ? 1 : 0;
}
// tied[j] = element j belongs to a group of size > 1 ; headidx[j] = j if head else 0 (for the max-scan)
__global__ void k_tied(const uint8_t* head, uint32_t n, uint8_t* tied, uint32_t* headidx) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if(j >= n) return;
	const bool single = head[j] && (j + 1 == n || head[j + 1]);
	tied[j] = single ? 0 : 1;
	headidx[j] = head[j] ? j : 0;
}
__global__ void k_gather_round(const uint64_t* t, uint64_t len, const uint64_t* pos, const uint32_t* idx, const uint32_t* gidfull,
                               uint32_t m, uint64_t d, uint64_t* key2, uint32_t* perm, uint32_t* gid) {
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if(u >= m) return;
	const uint32_t j = idx[u];
	key2[u] = suffix_key(t, len, pos[j], d);
	perm[u] = u; gid[u] = gidfull[j];
}
__global__ void k_gather_gid(const uint32_t* gid, const uint32_t* perm, uint32_t m, uint32_t* out) {
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if(u < m) out[u] = gid[perm[u]];
}
// after sorting by (gid, key2): element R[u] goes to slot idx[u]
__global__ void k_stage_round(const uint64_t* pos, const uint32_t* idx, const uint32_t* R, const uint64_t* key2, const uint32_t* gid,
                              uint32_t m, uint64_t* pos_tmp, uint8_t* newhead) {
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if(u >= m) return;
	const uint32_t r = R[u];
	pos_tmp[u] = pos[idx[r]];
	bool h = true;
	if(u > 0) { const uint32_t rp = R[u - 1]; h = gid[rp] != gid[r] || key2[rp] != key2[r]; }
	newhead[u] = h ? 1 : 0;
}
__global__ void k_commit_round(uint64_t* pos, uint8_t* head, const uint32_t* idx, const uint64_t* pos_tmp, const uint8_t* newhead, uint32_t m) {
	const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
	if(u >= m) return;
	const uint32_t j = idx[u];
	pos[j] = pos_tmp[u];
	if(newhead[u]) head[j] = 1;
}

struct OutArgs {
	const uint64_t* t; uint64_t len; const uint64_t* pos; uint32_t n; uint64_t row0;
	uint32_t* bwt_words;          // linear 2-bit BWT, 16 rows per u32, row r at bits 2*(r&15)
	uint32_t* sample;             // per 2^off_rate rows
	int off_rate;
	const uint64_t* frag_start; const uint32_t* frag_seq; uint32_t n_frag;
	const uint32_t* markbits; unsigned long long* n_bound; uint64_t* bound_row; uint64_t* bound_pos; uint32_t bound_cap;
	unsigned long long* zoff;
	unsigned long long* ftab_cnt; int ftab_chars;
};
__device__ __forceinline__ uint32_t seq_of(const OutArgs& a, uint64_t off) {
	uint32_t lo = 0, hi = a.n_frag;                 // last fragment with start <= off
	while(hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if(a.frag_start[mid] <= off) lo = mid; else hi = mid; }
	return a.frag_seq[lo];
}
__global__ void k_emit(const OutArgs a) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	const bool act = j < a.n;
	uint64_t suf = ~0ull;
	if(act) {
		const uint64_t p = a.pos[j], row = a.row0 + j;
		// BWT base (the '$' row is stored as A; Ebwt::buildToDisk bt2_idx.h:3570-3583)
		uint32_t c = 0;
		if(p == 0) *a.zoff = row; else c = (uint32_t)base_at(a.t, p - 1);
		if(c) atomicOr(&a.bwt_words[row >> 4], c << (2 * (row & 15)));
		// SA sample: sequence id of text position p+11 (clamped), bt2_idx.h:3647-3668
		if((row & ((1ull << a.off_rate) - 1)) == 0) {
			uint64_t adj = p + 11; if(adj >= a.len) adj = p; if(adj >= a.len) --adj;
			a.sample[row >> a.off_rate] = p > 0 ? seq_of(a, adj) : 0u;
		}
		if(a.markbits[p >> 5] & (1u << (p & 31))) {
			const unsigned long long k = atomicAdd(a.n_bound, 1ull);
			if(k < a.bound_cap) { a.bound_row[k] = row; a.bound_pos[k] = p; }
		}
		if(a.len - p >= (uint64_t)a.ftab_chars) suf = window32(a.t, p) >> (64 - 2 * a.ftab_chars);
	}
	// ftab histogram, warp-aggregated: rows are sorted so a warp sees one or two distinct prefixes
	const unsigned active = __ballot_sync(0xffffffffu, suf != ~0ull);
	if(suf != ~0ull) {
		const unsigned peers = __match_any_sync(active, suf);
		if((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&a.ftab_cnt[suf + 1], (unsigned long long)__popc(peers));
	}
}
// per-side base counts of the linear BWT (96 bytes = 24 u32 per side)
__global__ void k_side_counts(const uint32_t* bwt_words, uint64_t num_sides, uint64_t* cnt /*4*num_sides*/) {
	const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(s >= num_sides) return;
	uint64_t c1 = 0, c2 = 0, c3 = 0;
	for(int k = 0; k < 24; k++) {
		const uint32_t w = bwt_words[s * 24 + k];
		const uint32_t lo = w & 0x55555555u, hi = (w >> 1) & 0x55555555u;
		c1 += __popc(lo & ~hi); c2 += __popc(hi & ~lo); c3 += __popc(hi & lo);
	}
	cnt[s * 4 + 1] = c1; cnt[s * 4 + 2] = c2; cnt[s * 4 + 3] = c3; cnt[s * 4 + 0] = 384 - c1 - c2 - c3;
}
__global__ void k_assemble_sides(const uint32_t* bwt_words, const uint64_t* occ /*4*num_sides exclusive*/, uint64_t num_sides, uint32_t* sides /*32 u32 per side*/) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= num_sides * 32) return;
	const uint64_t s = i >> 5; const uint32_t k = (uint32_t)(i & 31);
	uint32_t v;
	if(k < 24) v = bwt_words[s * 24 + k];
	else { const uint64_t o = occ[s * 4 + ((k - 24) >> 1)]; v = (k & 1) ? (uint32_t)(o >> 32) : (uint32_t)o; }
	sides[i] = v;
}

// ---------------------------------------------------------------------------- host metadata
struct Meta {
	uint64_t len = 0, n_pat = 0, n_frag = 0;
	std::vector<uint64_t> plen, rstarts, frag_start; std::vector<uint32_t> frag_seq;
	std::vector<std::string> refnames;
	std::vector<uint64_t> mark_pos; std::vector<uint32_t> mark_idx;    // sorted by pos
};

struct Rec { uint64_t off, len; bool first; };

static inline int dnacat(int c) {        // asc2dnacat alphabet.cpp:36-58: 1 = ACGT, 2 = IUPAC/N, 3 = '-'
	switch(toupper(c)) {
		case 'A': case 'C': case 'G': case 'T': return 1;
		case 'B': case 'D': case 'H': case 'K': case 'M': case 'N': case 'R': case 'S': case 'V': case 'W': case 'X': case 'Y': return 2;
		case '-': return 3;
		default: return 0;
	}
}
static inline uint8_t dnacode(int c) { switch(toupper(c)) { case 'C': return 1; case 'G': return 2; case 'T': return 3; default: return 0; } }

// FASTA -> records + codes, following fastaRefReadSize/Append (ref_read.cpp:28-195)
static std::string read_fasta(const std::vector<std::string>& files, std::vector<Rec>& recs, std::vector<std::string>& names, std::vector<uint8_t>& codes) {
	for(size_t fi = 0; fi < files.size(); fi++) {
		FILE* f = fopen(files[fi].c_str(), "rb");
		if(!f) return "could not open FASTA file " + files[fi];
		std::vector<char> buf((size_t)1 << 24);
		std::string data; size_t k;
		while((k = fread(buf.data(), 1, buf.size(), f)) > 0) data.append(buf.data(), k);
		fclose(f);
		size_t p = 0; const size_t n = data.size();
		while(p < n && isspace((unsigned char)data[p])) p++;
		while(p < n) {
			if(data[p] != '>') return "reference file does not seem to be a FASTA file: " + files[fi];
			size_t e = p + 1; while(e < n && data[e] != '\n' && data[e] != '\r') e++;
			std::string name = data.substr(p + 1, e - p - 1);
			p = e;
			// sequence body up to the next '>' at any position (the reference scans characters, not lines)
			bool first = true; uint64_t off = 0, len = 0;
			while(p < n && data[p] != '>') {
				const int c = (unsigned char)data[p++];
				const int cat = dnacat(c);
				if(cat == 1) { codes.push_back(dnacode(c)); len++; }
				else if(cat >= 2) {
					if(len > 0) { Rec r = {off, len, first}; recs.push_back(r); first = false; off = 0; len = 0; }
					off++;
				}
			}
			if(len > 0 || off > 0 || first) { Rec r = {off, len, first}; recs.push_back(r); }
			// a name is kept only for sequences whose first record has bases (bt2_idx.h:3301-3318)
			bool has_first = false;
			for(size_t q = recs.size(); q-- > 0;) { if(recs[q].first) { has_first = recs[q].len > 0; break; } }
			if(has_first) names.push_back(name);
		}
	}
	return "";
}

static void build_meta(const std::vector<Rec>& recs, std::vector<std::string>& names, Meta& m) {
	m.n_pat = 0; m.n_frag = 0;
	for(size_t i = 0; i < recs.size(); i++) { if(recs[i].len > 0) m.n_frag++; if(recs[i].first && recs[i].len > 0) m.n_pat++; }
	m.plen.assign(m.n_pat, 0);
	long npat = -1;
	for(size_t i = 0; i < recs.size(); i++) {      // joinToDisk bt2_idx.h:3270-3284
		if(recs[i].first && recs[i].len > 0) { npat++; m.plen[npat] = recs[i].len + recs[i].off; }
		else if(npat >= 0) m.plen[npat] += recs[i].len + recs[i].off;
	}
	uint64_t seq = 0, off = 0, tot = 0;              // szsToDisk bt2_io.h:989-1030
	for(size_t i = 0; i < recs.size(); i++) {
		if(recs[i].len == 0) continue;
		if(recs[i].first) off = 0;
		off += recs[i].off;
		if(recs[i].first && recs[i].len > 0) seq++;
		m.rstarts.push_back(tot); m.rstarts.push_back(seq - 1); m.rstarts.push_back(off);
		m.frag_start.push_back(tot); m.frag_seq.push_back((uint32_t)(seq - 1));
		tot += recs[i].len; off += recs[i].len;
	}
	m.len = tot;
	for(size_t i = 0; i < names.size(); i++) if(names[i].empty()) { char b[32]; snprintf(b, sizeof b, "%zu", i); names[i] = b; }
	m.refnames = names;
	// boundary marks: joined offset of each sequence start minus 11 (bt2_idx.h:3508-3533); later sequences overwrite
	std::map<uint64_t, uint32_t> mk; uint64_t ro = 0; uint32_t idx = 0;
	for(size_t i = 0; i < recs.size(); i++) {
		if(recs[i].first && recs[i].len > 0) { const uint64_t o = ro < 11 ? 0 : ro - 11; mk[o] = idx++; }
		ro += recs[i].len;
	}
	for(std::map<uint64_t, uint32_t>::const_iterator it = mk.begin(); it != mk.end(); ++it) { m.mark_pos.push_back(it->first); m.mark_idx.push_back(it->second); }
}

static std::string get_uid(const std::string& h) {    // bt2_idx.h:2999-3009
	size_t nd = 0, j = 0;
	for(; j < h.size(); j++) { if(h[j] == ' ') break; if(h[j] == '|') nd++; if(nd == 2) break; }
	return h.substr(0, j);
}
static uint64_t get_tid(const std::string& s) {       // bt2_idx.h:3011-3030
	uint64_t t1 = 0, t2 = 0; bool dot = false;
	for(size_t i = 0; i < s.size(); i++) {
		if(s[i] == '.') { dot = true; continue; }
		const uint32_t num = (uint32_t)(s[i] - '0');
		if(dot) t2 = t2 * 10 + num; else t1 = t1 * 10 + num;
	}
	return t1 | (t2 << 32);
}
template <class T> static void put(FILE* f, T v) { fwrite(&v, sizeof(T), 1, f); }

static std::string write_cf3(const std::string& base, const Meta& m, const cfb_build_opts& o) {   // bt2_idx.h:1329-1506
	std::set<std::string> uids;
	for(size_t i = 0; i < m.refnames.size(); i++) uids.insert(get_uid(m.refnames[i]));
	std::map<std::string, uint64_t> u2t;
	{
		std::ifstream tf(o.conversion_table ? o.conversion_table : "");
		if(!tf.is_open()) return std::string("Error: ") + (o.conversion_table ? o.conversion_table : "(conversion table)") + " doesn't exist!";
		while(!tf.eof()) {
			std::string uid; tf >> uid;
			if(uid.empty() || uid[0] == '#') continue;
			std::string st; tf >> st;
			const uint64_t tid = get_tid(st);
			if(!uids.count(uid)) continue;
			if(u2t.count(uid)) continue;
			u2t[uid] = tid;
		}
	}
	FILE* f = fopen((base + ".3.cf").c_str(), "wb");
	if(!f) return "could not open " + base + ".3.cf for writing";
	std::set<uint64_t> tids;
	put<int32_t>(f, 1); put<uint64_t>(f, m.refnames.size());
	for(size_t i = 0; i < m.refnames.size(); i++) {
		const std::string uid = get_uid(m.refnames[i]);
		fwrite(uid.data(), 1, uid.size(), f); fputc(0, f);
		std::map<std::string, uint64_t>::const_iterator it = u2t.find(uid);
		if(it != u2t.end()) { put<uint64_t>(f, it->second); tids.insert(it->second); }
		else { fprintf(stderr, "Warning: taxonomy id doesn't exists for %s!\n", uid.c_str()); put<uint64_t>(f, 0); }
	}
	struct TN { uint64_t parent; uint8_t rank; };
	std::map<uint64_t, TN> tree;
	{
		std::ifstream tf(o.taxonomy_tree ? o.taxonomy_tree : "");
		if(!tf.is_open()) { fclose(f); return std::string("Error: ") + (o.taxonomy_tree ? o.taxonomy_tree : "(taxonomy tree)") + " doesn't exist!"; }
		std::string line;
		while(std::getline(tf, line)) {
			if(line.empty() || line[0] == '#') continue;
			std::istringstream cl(line); uint64_t tid = 0, par = 0; char dummy; std::string rk;
			cl >> tid >> dummy >> par >> dummy >> rk;
			if(tree.count(tid)) continue;
			TN t; t.parent = par; t.rank = (uint8_t)rank_from_name(rk.c_str()); tree[tid] = t;
		}
	}
	std::set<uint64_t> color;
	for(std::set<uint64_t>::const_iterator it = tids.begin(); it != tids.end(); ++it) {
		uint64_t tid = *it;
		while(tree.count(tid)) { const uint64_t par = tree[tid].parent; color.insert(tid); if(par == tid) break; tid = par; }
	}
	put<uint64_t>(f, color.size());
	for(std::set<uint64_t>::const_iterator it = color.begin(); it != color.end(); ++it) { put<uint64_t>(f, *it); put<uint64_t>(f, tree[*it].parent); put<uint16_t>(f, tree[*it].rank); }
	std::map<uint64_t, std::string> names;
	if(o.name_table && o.name_table[0]) {
		std::ifstream tf(o.name_table);
		if(!tf.is_open()) { fclose(f); return std::string("Error: ") + o.name_table + " doesn't exist!"; }
		std::string line;
		while(std::getline(tf, line)) {
			if(line.empty() || line[0] == '#') continue;
			if(line.find("scientific name") == std::string::npos) continue;
			std::istringstream cl(line); uint64_t tid = 0; char dummy; std::string nm;
			cl >> tid >> dummy >> nm;
			if(!color.count(tid)) continue;
			std::string tmp;
			while(cl >> tmp) { if(tmp == "|") break; nm.push_back('@'); nm += tmp; }
			names[tid] = nm;
		}
	}
	put<uint64_t>(f, names.size());
	for(std::map<uint64_t, std::string>::const_iterator it = names.begin(); it != names.end(); ++it) { put<uint64_t>(f, it->first); fwrite(it->second.data(), 1, it->second.size(), f); fputc('\n', f); }
	std::map<uint64_t, uint64_t> sizes;
	for(size_t i = 0; i < m.refnames.size(); i++) {
		std::map<std::string, uint64_t>::const_iterator it = u2t.find(get_uid(m.refnames[i]));
		if(it == u2t.end()) continue;
		sizes[it->second] += m.plen[i];
	}
	if(o.size_table && o.size_table[0]) {
		std::ifstream tf(o.size_table);
		if(!tf.is_open()) { fclose(f); return std::string("Error: ") + o.size_table + " doesn't exist!"; }
		while(!tf.eof()) { std::string st; tf >> st; if(st.empty() || st[0] == '#') continue; uint64_t sz = 0; tf >> sz; sizes[get_tid(st)] = sz; }
	}
	put<uint64_t>(f, sizes.size());
	for(std::map<uint64_t, uint64_t>::const_iterator it = sizes.begin(); it != sizes.end(); ++it) { put<uint64_t>(f, it->first); put<uint64_t>(f, it->second); }
	fclose(f);
	return "";
}

}  // namespace

extern "C" const char* cfb_build_last_error(void) { return g_berr.c_str(); }

extern "C" void cfb_build_opts_default(cfb_build_opts* o) {
	if(!o) return;
	memset(o, 0, sizeof *o); o->ftab_chars = 10; o->off_rate = 4; o->synth_div = 0.03; o->device = 0;
}

extern "C" int cfb_build_index(const cfb_build_opts* o) {
	if(!o || !o->out_base) return bfail(CFB_EINVAL, "cfb_build_index: null options / output base");
	if(o->ftab_chars < 1 || o->ftab_chars > 14 || o->off_rate < 0 || o->off_rate > 16) return bfail(CFB_EINVAL, "unsupported ftab_chars/off_rate");
	int ndev = 0;
	if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= o->device) return bfail(CFB_ENODEV, "no CUDA device %d; the index builder runs on the GPU only", o->device);
	BCK(cudaSetDevice(o->device));
	const std::string base = o->out_base;
	const bool synth = o->n_fasta == 0;
	Meta m; std::vector<uint8_t> codes;
	SynthSpec sp; memset(&sp, 0, sizeof sp);
	if(synth) {
		if(o->synth_genera < 1 || o->synth_species < 1 || o->synth_len < 32) return bfail(CFB_EINVAL, "synthetic spec needs genera, species >= 1 and len >= 32");
		sp.genera = o->synth_genera; sp.species = o->synth_species; sp.len = o->synth_len; sp.seed = o->synth_seed;
		sp.div_q32 = (uint32_t)std::min(4294967295.0, o->synth_div * 4294967296.0);
		std::vector<Rec> recs; std::vector<std::string> names;
		const uint32_t ns = sp.genera * sp.species;
		for(uint32_t i = 0; i < ns; i++) { Rec r = {0, sp.len, true}; recs.push_back(r); char b[64]; snprintf(b, sizeof b, "%.40s%u", o->synth_prefix ? o->synth_prefix : "seq", i); names.push_back(b); }
		build_meta(recs, names, m);
	} else {
		std::vector<std::string> files; for(int i = 0; i < o->n_fasta; i++) files.push_back(o->fasta[i]);
		std::vector<Rec> recs; std::vector<std::string> names;
		std::string e = read_fasta(files, recs, names, codes);
		if(!e.empty()) return bfail(CFB_EIO, "%s", e.c_str());
		build_meta(recs, names, m);
		if(m.len != codes.size()) return bfail(CFB_EIO, "internal: joined length mismatch");
	}
	if(m.len < 1 || m.n_pat < 1) return bfail(CFB_EIO, "reference is empty");
	const uint64_t len = m.len;
	if(o->verbose) fprintf(stderr, "[cfb-build] joined length %llu, %llu sequences, %llu fragments\n", (unsigned long long)len, (unsigned long long)m.n_pat, (unsigned long long)m.n_frag);
	{ std::string e = write_cf3(base, m, *o); if(!e.empty()) return bfail(CFB_EIO, "%s", e.c_str()); }

	// ---- geometry (EbwtParams::init bt2_idx.h:133-167), lineRate fixed at 7
	const uint64_t bwt_len = len + 1, side_bwt_sz = 96, num_sides = (len / 4 + 1 + side_bwt_sz - 1) / side_bwt_sz;
	const uint64_t ftab_len = ((uint64_t)1 << (2 * o->ftab_chars)) + 1, eftab_len = 2 * (uint64_t)o->ftab_chars;
	const uint64_t offs_len = (bwt_len + ((uint64_t)1 << o->off_rate) - 1) >> o->off_rate;
	const bool wide = m.n_pat > 65535;

	// ---- text on the device
	const uint64_t nwords = (len + 31) / 32 + 4;
	DBuf<uint64_t> text; BCK(text.alloc(nwords)); BCK(cudaMemset(text.p, 0, nwords * 8));
	if(synth) { k_synth_text<<<(unsigned)((nwords + 255) / 256), 256>>>(sp, text.p, (len + 31) / 32, len); }
	else {
		DBuf<uint8_t> dc; BCK(dc.alloc(len)); BCK(cudaMemcpy(dc.p, codes.data(), len, cudaMemcpyHostToDevice));
		k_pack_text<<<(unsigned)(((len + 31) / 32 + 255) / 256), 256>>>(dc.p, len, text.p, (len + 31) / 32);
		BCK(cudaDeviceSynchronize());
		std::vector<uint8_t>().swap(codes);
	}
	BCK(cudaDeviceSynchronize());

	// ---- global outputs
	DBuf<uint32_t> bwt; BCK(bwt.alloc(num_sides * 24)); BCK(cudaMemset(bwt.p, 0, num_sides * 24 * 4));
	DBuf<uint32_t> sample; BCK(sample.alloc(offs_len)); BCK(cudaMemset(sample.p, 0, offs_len * 4));
	DBuf<unsigned long long> ftab_cnt; BCK(ftab_cnt.alloc(ftab_len + 1)); BCK(cudaMemset(ftab_cnt.p, 0, (ftab_len + 1) * 8));
	DBuf<uint32_t> markbits; BCK(markbits.alloc(len / 32 + 2)); BCK(cudaMemset(markbits.p, 0, (len / 32 + 2) * 4));
	{
		std::vector<uint32_t> hb(len / 32 + 2, 0);
		for(size_t i = 0; i < m.mark_pos.size(); i++) hb[m.mark_pos[i] >> 5] |= 1u << (m.mark_pos[i] & 31);
		BCK(cudaMemcpy(markbits.p, hb.data(), hb.size() * 4, cudaMemcpyHostToDevice));
	}
	const uint32_t bound_cap = (uint32_t)m.mark_pos.size() + 16;
	DBuf<uint64_t> bound_row, bound_pos; BCK(bound_row.alloc(bound_cap)); BCK(bound_pos.alloc(bound_cap));
	DBuf<unsigned long long> scal; BCK(scal.alloc(32)); BCK(cudaMemset(scal.p, 0, 32 * 8));   // [0..15] hist, [16] n_bound, [17] zoff, [18] select count
	DBuf<uint64_t> d_frag_start; DBuf<uint32_t> d_frag_seq;
	BCK(d_frag_start.alloc(m.frag_start.size())); BCK(d_frag_seq.alloc(m.frag_seq.size()));
	BCK(cudaMemcpy(d_frag_start.p, m.frag_start.data(), m.frag_start.size() * 8, cudaMemcpyHostToDevice));
	BCK(cudaMemcpy(d_frag_seq.p, m.frag_seq.data(), m.frag_seq.size() * 4, cudaMemcpyHostToDevice));

	// ---- bucket sizes
	k_bucket_hist<<<1184, 256>>>(text.p, len, scal.p);
	unsigned long long hist[16];
	BCK(cudaMemcpy(hist, scal.p, sizeof hist, cudaMemcpyDeviceToHost));
	uint64_t maxb = 0; for(int b = 0; b < 16; b++) maxb = std::max<uint64_t>(maxb, hist[b]);
	if(maxb >= (1ull << 31)) return bfail(CFB_ENOMEM, "largest 2-mer bucket has %llu suffixes (limit 2^31): reference too large or too skewed for this builder", (unsigned long long)maxb);
	const uint32_t cap = (uint32_t)maxb + 1;

	// ---- per-bucket workspace
	DBuf<uint64_t> pos, pos_alt, key, key_alt, key2, key2_alt, pos_tmp;
	DBuf<uint8_t> head, tied, newhead;
	DBuf<uint32_t> headidx, gidfull, idx, perm, perm_alt, gid, gid_s, gid_s_alt;
	BCK(pos.alloc(cap)); BCK(pos_alt.alloc(cap)); BCK(key.alloc(cap)); BCK(key_alt.alloc(cap));
	BCK(head.alloc(cap)); BCK(tied.alloc(cap)); BCK(headidx.alloc(cap)); BCK(gidfull.alloc(cap)); BCK(idx.alloc(cap));
	size_t tmp_bytes = 0, tb = 0;
	{
		cub::DoubleBuffer<uint64_t> dk(key.p, key_alt.p), dv(pos.p, pos_alt.p);
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)cap, 0, 64); tmp_bytes = std::max(tmp_bytes, tb);
		cub::DoubleBuffer<uint64_t> dk2(key.p, key_alt.p); cub::DoubleBuffer<uint32_t> dp(idx.p, idx.p);
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dk2, dp, (int)cap, 0, 64); tmp_bytes = std::max(tmp_bytes, tb);
		cub::DoubleBuffer<uint32_t> dg(idx.p, idx.p);
		cub::DeviceRadixSort::SortPairs(nullptr, tb, dg, dp, (int)cap, 0, 32); tmp_bytes = std::max(tmp_bytes, tb);
		cub::CountingInputIterator<uint64_t> cit(0);
		InBucket pr; pr.t = text.p; pr.len = len; pr.b = 0;
		cub::DeviceSelect::If(nullptr, tb, cit, pos.p, (unsigned long long*)scal.p, (int)(1 << 30), pr); tmp_bytes = std::max(tmp_bytes, tb);
		cub::CountingInputIterator<uint32_t> c32(0);
		cub::DeviceSelect::Flagged(nullptr, tb, c32, tied.p, idx.p, (unsigned long long*)scal.p, (int)cap); tmp_bytes = std::max(tmp_bytes, tb);
		cub::DeviceScan::InclusiveScan(nullptr, tb, headidx.p, gidfull.p, cub::Max(), (int)cap); tmp_bytes = std::max(tmp_bytes, tb);
	}
	DBuf<uint8_t> tmp; BCK(tmp.alloc(tmp_bytes + 256));
	bool round_ws = false;       // refinement buffers are allocated on first use (sized by the first tie count)
	uint32_t round_cap = 0;

	uint64_t row0 = 0;           // the empty suffix is the LAST row (row len): '$' sorts after every base
	int max_rounds = 0;
	for(int b = 0; b < 16; b++) {
		const uint32_t n = (uint32_t)hist[b];
		if(n == 0) continue;
		// (1) positions of this bucket, in chunks of 2^30 text positions
		uint64_t got = 0;
		for(uint64_t c0 = 0; c0 < len; c0 += (1ull << 30)) {
			const uint64_t cn = std::min<uint64_t>(1ull << 30, len - c0);
			cub::CountingInputIterator<uint64_t> cit(c0);
			InBucket pr; pr.t = text.p; pr.len = len; pr.b = b;
			size_t tbb = tmp_bytes;
			BCK(cub::DeviceSelect::If(tmp.p, tbb, cit, pos.p + got, (unsigned long long*)(scal.p + 18), (int)cn, pr));
			unsigned long long k = 0; BCK(cudaMemcpy(&k, scal.p + 18, 8, cudaMemcpyDeviceToHost));
			got += k;
		}
		if(got != n) return bfail(CFB_ECUDA, "internal: bucket %d selected %llu of %u suffixes", b, (unsigned long long)got, n);
		const unsigned gb = (n + 255) / 256;
		// (2) first window after the 2-base bucket prefix, sort, group heads
		k_keys<<<gb, 256>>>(text.p, len, pos.p, n, 2, key.p);
		{
			cub::DoubleBuffer<uint64_t> dk(key.p, key_alt.p), dv(pos.p, pos_alt.p);
			size_t tbb = tmp_bytes;
			BCK(cub::DeviceRadixSort::SortPairs(tmp.p, tbb, dk, dv, (int)n, 0, 64));
			if(dk.Current() != key.p) std::swap(key.p, key_alt.p);
			if(dv.Current() != pos.p) std::swap(pos.p, pos_alt.p);
		}
		k_heads<<<gb, 256>>>(key.p, n, head.p);
		// (3) refine tied groups window by window
		uint64_t d = 2 + kWin; int rounds = 0;
		for(;;) {
			k_tied<<<gb, 256>>>(head.p, n, tied.p, headidx.p);
			cub::CountingInputIterator<uint32_t> c32(0);
			size_t tbb = tmp_bytes;
			BCK(cub::DeviceSelect::Flagged(tmp.p, tbb, c32, tied.p, idx.p, (unsigned long long*)(scal.p + 18), (int)n));
			unsigned long long mm = 0; BCK(cudaMemcpy(&mm, scal.p + 18, 8, cudaMemcpyDeviceToHost));
			if(mm == 0) break;
			const uint32_t mcnt = (uint32_t)mm;
			if(!round_ws || mcnt > round_cap) {
				round_cap = std::max<uint32_t>(mcnt + mcnt / 8 + 1024, round_cap);
				BCK(key2.alloc(round_cap)); BCK(key2_alt.alloc(round_cap)); BCK(pos_tmp.alloc(round_cap)); BCK(newhead.alloc(round_cap));
				BCK(perm.alloc(round_cap)); BCK(perm_alt.alloc(round_cap)); BCK(gid.alloc(round_cap)); BCK(gid_s.alloc(round_cap)); BCK(gid_s_alt.alloc(round_cap));
				round_ws = true;
			}
			tbb = tmp_bytes;
			BCK(cub::DeviceScan::InclusiveScan(tmp.p, tbb, headidx.p, gidfull.p, cub::Max(), (int)n));
			const unsigned mb = (mcnt + 255) / 256;
			k_gather_round<<<mb, 256>>>(text.p, len, pos.p, idx.p, gidfull.p, mcnt, d, key2.p, perm.p, gid.p);
			// keys in slot order must survive the sort: sort a copy
			BCK(cudaMemcpy(key2_alt.p, key2.p, (size_t)mcnt * 8, cudaMemcpyDeviceToDevice));
			{   // stable sort by window key ...
				cub::DoubleBuffer<uint64_t> dk(key2_alt.p, pos_tmp.p); cub::DoubleBuffer<uint32_t> dv(perm.p, perm_alt.p);
				tbb = tmp_bytes;
				BCK(cub::DeviceRadixSort::SortPairs(tmp.p, tbb, dk, dv, (int)mcnt, 0, 64));
				if(dv.Current() != perm.p) std::swap(perm.p, perm_alt.p);
			}
			k_gather_gid<<<mb, 256>>>(gid.p, perm.p, mcnt, gid_s.p);
			{   // ... then stable sort by group id
				int bits = 1; while((1ull << bits) < n) bits++;
				cub::DoubleBuffer<uint32_t> dk(gid_s.p, gid_s_alt.p), dv(perm.p, perm_alt.p);
				tbb = tmp_bytes;
				BCK(cub::DeviceRadixSort::SortPairs(tmp.p, tbb, dk, dv, (int)mcnt, 0, bits));
				if(dv.Current() != perm.p) std::swap(perm.p, perm_alt.p);
			}
			k_stage_round<<<mb, 256>>>(pos.p, idx.p, perm.p, key2.p, gid.p, mcnt, pos_tmp.p, newhead.p);
			k_commit_round<<<mb, 256>>>(pos.p, head.p, idx.p, pos_tmp.p, newhead.p, mcnt);
			d += kWin; rounds++;
			if(d > len + 64) break;      // cannot happen for distinct suffixes; guards against bugs
		}
		max_rounds = std::max(max_rounds, rounds);
		// (4) emit everything derived from this slice of the suffix array
		OutArgs oa; oa.t = text.p; oa.len = len; oa.pos = pos.p; oa.n = n; oa.row0 = row0; oa.bwt_words = bwt.p; oa.sample = sample.p; oa.off_rate = o->off_rate;
		oa.frag_start = d_frag_start.p; oa.frag_seq = d_frag_seq.p; oa.n_frag = (uint32_t)m.frag_start.size();
		oa.markbits = markbits.p; oa.n_bound = scal.p + 16; oa.bound_row = bound_row.p; oa.bound_pos = bound_pos.p; oa.bound_cap = bound_cap;
		oa.zoff = scal.p + 17; oa.ftab_cnt = ftab_cnt.p; oa.ftab_chars = o->ftab_chars;
		k_emit<<<(n + 255) / 256 * 1, 256>>>(oa);
		BCK(cudaDeviceSynchronize());
		row0 += n;
		if(o->verbose) fprintf(stderr, "[cfb-build] bucket %d: %u suffixes, %d refinement rounds\n", b, n, rounds);
	}
	if(row0 != len) return bfail(CFB_ECUDA, "internal: emitted %llu of %llu rows", (unsigned long long)row0, (unsigned long long)len);

	// ---- last row (empty suffix, saElt == len): BWT base = text[len-1]; sample = seq of text position len-1
	uint8_t tail[64]; const uint64_t tail_n = std::min<uint64_t>(len, 40);
	{
		std::vector<uint64_t> tw((tail_n + 31) / 32 + 2);
		const uint64_t w0 = (len - tail_n) >> 5;
		BCK(cudaMemcpy(tw.data(), text.p + w0, tw.size() * 8, cudaMemcpyDeviceToHost));
		for(uint64_t k = 0; k < tail_n; k++) { const uint64_t i = len - tail_n + k; tail[k] = (uint8_t)((tw[(i >> 5) - w0] >> (62 - 2 * (i & 31))) & 3); }
	}
	{
		const uint32_t c = tail[tail_n - 1];
		uint32_t wv = 0; BCK(cudaMemcpy(&wv, bwt.p + (len >> 4), 4, cudaMemcpyDeviceToHost)); wv |= c << (2 * (len & 15)); BCK(cudaMemcpy(bwt.p + (len >> 4), &wv, 4, cudaMemcpyHostToDevice));
		if((len & ((1ull << o->off_rate) - 1)) == 0) { const uint32_t s0 = m.frag_seq.back(); BCK(cudaMemcpy(sample.p + (len >> o->off_rate), &s0, 4, cudaMemcpyHostToDevice)); }
	}

	// ---- sides: per-side counts -> exclusive occ, '$' not counted as A
	unsigned long long zoff = 0, nbound = 0;
	BCK(cudaMemcpy(&nbound, scal.p + 16, 8, cudaMemcpyDeviceToHost)); BCK(cudaMemcpy(&zoff, scal.p + 17, 8, cudaMemcpyDeviceToHost));
	DBuf<uint64_t> cnt; BCK(cnt.alloc(num_sides * 4));
	k_side_counts<<<(unsigned)((num_sides + 255) / 256), 256>>>(bwt.p, num_sides, cnt.p);
	std::vector<uint64_t> hcnt(num_sides * 4);
	BCK(cudaMemcpy(hcnt.data(), cnt.p, hcnt.size() * 8, cudaMemcpyDeviceToHost));
	hcnt[(zoff / 384) * 4 + 0] -= 1;                       // the '$' looks like an A but is not counted
	uint64_t run[4] = {0, 0, 0, 0}, tot[4] = {0, 0, 0, 0};
	for(uint64_t s = 0; s < num_sides; s++) for(int c = 0; c < 4; c++) { const uint64_t v = hcnt[s * 4 + c]; hcnt[s * 4 + c] = run[c]; run[c] += v; }
	for(int c = 0; c < 4; c++) tot[c] = run[c];
	// padding rows past the end of the BWT were counted as A in the last side only: they do not affect any stored occ
	tot[0] -= (num_sides * 384 - bwt_len);
	BCK(cudaMemcpy(cnt.p, hcnt.data(), hcnt.size() * 8, cudaMemcpyHostToDevice));
	DBuf<uint32_t> sides; BCK(sides.alloc(num_sides * 32));
	k_assemble_sides<<<(unsigned)((num_sides * 32 + 255) / 256), 256>>>(bwt.p, cnt.p, num_sides, sides.p);
	BCK(cudaDeviceSynchronize());

	// ---- ftab / eftab on the host (bt2_idx.h:3585-3612,3775-3815)
	std::vector<uint64_t> ftab(ftab_len);
	{ std::vector<unsigned long long> fc(ftab_len + 1); BCK(cudaMemcpy(fc.data(), ftab_cnt.p, (ftab_len + 1) * 8, cudaMemcpyDeviceToHost)); for(uint64_t i = 0; i < ftab_len; i++) ftab[i] = fc[i]; }
	std::vector<uint8_t> absorb(ftab_len, 0);
	{
		// suffixes shorter than ftabChars sort after every longer suffix sharing their bases: the next long
		// suffix in order is the first one whose prefix exceeds the short suffix padded with T's
		const int fc = o->ftab_chars;
		std::vector<std::pair<uint64_t, int> > shorts;       // (first prefix value strictly after the suffix, -length)
		for(int L = 0; L < fc && (uint64_t)L <= len; L++) {
			uint64_t v = 0; for(int k = 0; k < L; k++) v = (v << 2) | tail[tail_n - L + k];
			const int padb = 2 * (fc - L);
			const uint64_t after = ((v << padb) | ((1ull << padb) - 1)) + 1;
			shorts.push_back(std::make_pair(after, -L));
		}
		std::sort(shorts.begin(), shorts.end());
		size_t i = 0;
		while(i < shorts.size()) {
			uint64_t x = shorts[i].first;                        // candidate sufInt of the next long suffix
			while(x + 1 < ftab_len && ftab[x + 1] == 0) x++;
			size_t j = i; uint8_t cntv = 0;
			while(j < shorts.size()) {
				uint64_t y = shorts[j].first; while(y + 1 < ftab_len && ftab[y + 1] == 0) y++;
				if(y != x) break;
				cntv++; j++;
			}
			if(x + 1 >= ftab_len) absorb[ftab_len - 1] = cntv; else absorb[x] = cntv;
			i = j;
		}
	}
	std::vector<uint64_t> eftab(eftab_len, 0);
	{
		uint64_t ecur = 0;
		for(uint64_t i = 1; i < ftab_len; i++) {
			const uint64_t prev = ftab[i - 1] <= len ? ftab[i - 1] : eftab[(ftab[i - 1] ^ ~0ull) * 2 + 1];
			const uint64_t lo = ftab[i] + prev;
			if(absorb[i] > 0) { const uint64_t hi = lo + absorb[i]; eftab[ecur * 2] = lo; eftab[ecur * 2 + 1] = hi; ftab[i] = (ecur++) ^ ~0ull; }
			else ftab[i] = lo;
		}
	}
	uint64_t fchr[5] = {0, tot[0], tot[0] + tot[1], tot[0] + tot[1] + tot[2], len};

	// ---- write .1.cf / .2.cf / .4.cf
	{
		FILE* f = fopen((base + ".1.cf").c_str(), "wb");
		if(!f) return bfail(CFB_EIO, "could not open %s.1.cf for writing", base.c_str());
		put<int32_t>(f, 1); put<uint64_t>(f, len); put<int32_t>(f, 7); put<int32_t>(f, 2); put<int32_t>(f, o->off_rate); put<int32_t>(f, o->ftab_chars); put<int32_t>(f, -1);
		put<uint64_t>(f, m.n_pat); fwrite(m.plen.data(), 8, m.plen.size(), f);
		put<uint64_t>(f, m.n_frag); fwrite(m.rstarts.data(), 8, m.rstarts.size(), f);
		std::vector<uint32_t> hs((size_t)1 << 24);
		for(uint64_t o0 = 0; o0 < num_sides * 32; o0 += hs.size()) {
			const uint64_t k = std::min<uint64_t>(hs.size(), num_sides * 32 - o0);
			BCK(cudaMemcpy(hs.data(), sides.p + o0, k * 4, cudaMemcpyDeviceToHost));
			fwrite(hs.data(), 4, k, f);
		}
		put<uint64_t>(f, zoff);
		fwrite(fchr, 8, 5, f); fwrite(ftab.data(), 8, ftab.size(), f); fwrite(eftab.data(), 8, eftab.size(), f);
		for(size_t i = 0; i < m.refnames.size(); i++) { fwrite(m.refnames[i].data(), 1, m.refnames[i].size(), f); fputc('\n', f); }
		fputc(0, f);
		if(fclose(f) != 0) return bfail(CFB_EIO, "error writing %s.1.cf", base.c_str());
	}
	{
		FILE* f = fopen((base + ".2.cf").c_str(), "wb");
		if(!f) return bfail(CFB_EIO, "could not open %s.2.cf for writing", base.c_str());
		put<int32_t>(f, 1);
		std::vector<uint32_t> hs((size_t)1 << 24); std::vector<uint16_t> h16;
		for(uint64_t o0 = 0; o0 < offs_len; o0 += hs.size()) {
			const uint64_t k = std::min<uint64_t>(hs.size(), offs_len - o0);
			BCK(cudaMemcpy(hs.data(), sample.p + o0, k * 4, cudaMemcpyDeviceToHost));
			if(wide) fwrite(hs.data(), 4, k, f);
			else { h16.resize(k); for(uint64_t q = 0; q < k; q++) h16[q] = (uint16_t)hs[q]; fwrite(h16.data(), 2, k, f); }
		}
		if(fclose(f) != 0) return bfail(CFB_EIO, "error writing %s.2.cf", base.c_str());
	}
	{
		std::vector<uint64_t> br(nbound), bp(nbound);
		if(nbound > bound_cap) return bfail(CFB_ECUDA, "internal: boundary overflow");
		BCK(cudaMemcpy(br.data(), bound_row.p, nbound * 8, cudaMemcpyDeviceToHost)); BCK(cudaMemcpy(bp.data(), bound_pos.p, nbound * 8, cudaMemcpyDeviceToHost));
		std::map<uint64_t, uint32_t> bm;
		for(uint64_t i = 0; i < nbound; i++) {
			const size_t k = std::lower_bound(m.mark_pos.begin(), m.mark_pos.end(), bp[i]) - m.mark_pos.begin();
			bm[br[i]] = m.mark_idx[k];
		}
		FILE* f = fopen((base + ".4.cf").c_str(), "wb");
		if(!f) return bfail(CFB_EIO, "could not open %s.4.cf for writing", base.c_str());
		put<int32_t>(f, 1); put<uint64_t>(f, bm.size());
		for(std::map<uint64_t, uint32_t>::const_iterator it = bm.begin(); it != bm.end(); ++it) { put<uint64_t>(f, it->first); put<uint32_t>(f, it->second); }
		fclose(f);
	}
	if(o->verbose) fprintf(stderr, "[cfb-build] done: %llu sides, max %d refinement rounds\n", (unsigned long long)num_sides, max_rounds);
	return CFB_OK;
}

// ---------------------------------------------------------------------------- synthetic reads
__global__ void k_synth_reads(SynthSpec sp, uint64_t n, uint32_t rdlen, uint64_t seed, uint8_t* out) {
	const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(r >= n) return;
	const uint64_t h0 = mix64(seed * 0x9E3779B97F4A7C15ull + r);
	uint8_t* o = out + r * rdlen;
	const bool random = (h0 & 0xffff) < 3277;                 // 5% reads of random sequence
	const uint32_t nseq = sp.genera * sp.species;
	const uint32_t seq = (uint32_t)((h0 >> 16) % nseq);
	const uint64_t pos = mix64(h0 ^ 0x1234) % (sp.len - rdlen + 1);
	const bool rc = (mix64(h0 ^ 0x77) & 1) != 0;
	for(uint32_t i = 0; i < rdlen; i++) {
		const uint64_t hi = mix64(h0 + 0x51ED27ull * (i + 1));
		int c;
		if(random) c = (int)(hi & 3);
		else {
			c = synth_base(sp, seq, pos + i);
			if(((hi >> 8) & 0xffff) < 655) c = (c + 1) & 3;     // 1% substitutions
		}
		if(((hi >> 32) & 0xffff) < 66) c = 4;                  // 0.1% N
		if(rc && !random) { o[rdlen - 1 - i] = (uint8_t)(c > 3 ? 4 : 3 - c); } else o[i] = (uint8_t)c;
	}
}

extern "C" int cfb_synth_reads(const cfb_build_opts* o, uint64_t n, uint32_t rdlen, uint64_t read_seed, uint8_t* out_codes) {
	if(!o || !out_codes || rdlen == 0 || o->synth_len < rdlen) return bfail(CFB_EINVAL, "cfb_synth_reads: bad arguments");
	BCK(cudaSetDevice(o->device));
	SynthSpec sp; sp.genera = o->synth_genera; sp.species = o->synth_species; sp.len = o->synth_len; sp.seed = o->synth_seed;
	sp.div_q32 = (uint32_t)std::min(4294967295.0, o->synth_div * 4294967296.0);
	DBuf<uint8_t> d; BCK(d.alloc(n * rdlen));
	k_synth_reads<<<(unsigned)((n + 127) / 128), 128>>>(sp, n, rdlen, read_seed, d.p);
	BCK(cudaMemcpy(out_codes, d.p, n * rdlen, cudaMemcpyDeviceToHost));
	return CFB_OK;
}

// Paired / mixed-length variant of the same recipe (SURVEY.md 8d: 2 x L PE with insert U[ins_lo, ins_hi] and mate 2 reverse-
// complemented; U[len_lo, len_hi] read lengths).  codes: mate-major (mates, n, len_hi), rows padded with N; lens: (mates, n).
__global__ void k_synth_reads_ex(SynthSpec sp, cfb_synth_read_opts ro, uint64_t n, uint64_t seed, uint8_t* out, uint32_t* lens) {
	const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(r >= n) return;
	const uint64_t h0 = mix64(seed * 0x9E3779B97F4A7C15ull + r);
	const bool random = (h0 & 0xffff) < 3277;                 // 5% units of random sequence
	const uint32_t nseq = sp.genera * sp.species;
	const uint32_t seq = (uint32_t)((h0 >> 16) % nseq);
	const bool rc = (mix64(h0 ^ 0x77) & 1) != 0;
	const uint32_t span = ro.len_hi - ro.len_lo + 1;
	const int mates = ro.paired ? 2 : 1;
	uint32_t L[2]; L[0] = ro.len_lo + (uint32_t)(mix64(h0 ^ 0xA1) % span); L[1] = ro.paired ? ro.len_lo + (uint32_t)(mix64(h0 ^ 0xA2) % span) : 0;
	uint64_t frag = L[0];
	if(ro.paired) { frag = ro.ins_lo + mix64(h0 ^ 0xA3) % (ro.ins_hi - ro.ins_lo + 1); if(frag < L[0]) frag = L[0]; if(frag < L[1]) frag = L[1]; }
	if(frag > sp.len) frag = sp.len;
	for(int m = 0; m < mates; m++) if(L[m] > frag) L[m] = (uint32_t)frag;
	const uint64_t pos = mix64(h0 ^ 0x1234) % (sp.len - frag + 1);
	// fragment base at offset q of the sequenced strand (the reverse strand reads the genome backwards, complemented)
	auto frag_base = [&](uint64_t q) -> int { if(!rc) return synth_base(sp, seq, pos + q); return 3 - synth_base(sp, seq, pos + frag - 1 - q); };
	for(int m = 0; m < mates; m++) {
		uint8_t* o = out + ((uint64_t)m * n + r) * ro.len_hi;
		lens[(uint64_t)m * n + r] = L[m];
		for(uint32_t i = 0; i < ro.len_hi; i++) {
			int c = 4;
			if(i < L[m]) {
				const uint64_t hi = mix64(h0 + 0x51ED27ull * (i + 1) + 0x9E37ull * (m + 1));
				if(random) c = (int)(hi & 3);
				else {
					c = m == 0 ? frag_base(i) : 3 - frag_base(frag - 1 - i);       // mate 2: reverse complement of the fragment's far end
					if(((hi >> 8) & 0xffff) < 655) c = (c + 1) & 3;          // 1% substitutions
				}
				if(((hi >> 32) & 0xffff) < 66) c = 4;                       // 0.1% N
			}
			o[i] = (uint8_t)c;
		}
	}
}
extern "C" int cfb_synth_reads_ex(const cfb_build_opts* o, const cfb_synth_read_opts* ro, uint64_t n, uint64_t read_seed, uint8_t* out_codes, uint32_t* out_lens) {
	if(!o || !ro || !out_codes || !out_lens || ro->len_lo < 1 || ro->len_hi < ro->len_lo || o->synth_len < ro->len_hi || (ro->paired && (ro->ins_hi < ro->ins_lo || ro->ins_hi > o->synth_len)))
		return bfail(CFB_EINVAL, "cfb_synth_reads_ex: bad arguments");
	BCK(cudaSetDevice(o->device));
	SynthSpec sp; sp.genera = o->synth_genera; sp.species = o->synth_species; sp.len = o->synth_len; sp.seed = o->synth_seed;
	sp.div_q32 = (uint32_t)std::min(4294967295.0, o->synth_div * 4294967296.0);
	const uint64_t mates = ro->paired ? 2 : 1;
	DBuf<uint8_t> d; BCK(d.alloc(n * mates * ro->len_hi)); DBuf<uint32_t> dl; BCK(dl.alloc(n * mates));
	k_synth_reads_ex<<<(unsigned)((n + 127) / 128), 128>>>(sp, *ro, n, read_seed, d.p, dl.p);
	BCK(cudaMemcpy(out_codes, d.p, n * mates * ro->len_hi, cudaMemcpyDeviceToHost));
	BCK(cudaMemcpy(out_lens, dl.p, n * mates * 4, cudaMemcpyDeviceToHost));
	return CFB_OK;
}

// Materialise the synthetic genomes as FASTA (tests: byte-compare this builder with centrifuge-build-bin).
extern "C" int cfb_synth_fasta(const cfb_build_opts* o, const char* path) {
	if(!o || !path) return bfail(CFB_EINVAL, "null argument");
	SynthSpec sp; sp.genera = o->synth_genera; sp.species = o->synth_species; sp.len = o->synth_len; sp.seed = o->synth_seed;
	sp.div_q32 = (uint32_t)std::min(4294967295.0, o->synth_div * 4294967296.0);
	FILE* f = fopen(path, "wb");
	if(!f) return bfail(CFB_EIO, "cannot write %s", path);
	std::string line;
	for(uint32_t s = 0; s < sp.genera * sp.species; s++) {
		fprintf(f, ">%.40s%u\n", o->synth_prefix ? o->synth_prefix : "seq", s);
		for(uint64_t p = 0; p < sp.len; p += 80) {
			line.clear();
			for(uint64_t q = p; q < std::min(sp.len, p + 80); q++) line.push_back("ACGT"[synth_base(sp, s, q)]);
			line.push_back('\n'); fwrite(line.data(), 1, line.size(), f);
		}
	}
	fclose(f);
	return CFB_OK;
}
