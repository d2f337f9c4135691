// cf_gunzip.cu -- gzip (RFC 1952) inflater on the device: the cfb_gunzip_* entry points of include/cfb200.h.
//
// A member's DEFLATE stream is decoded in passes over a span of compressed bytes (at most kMaxChunks chunks).  Chunk 0
// of a pass starts from the known state carried over from the previous pass; every other chunk searches its first
// bits for a block header (k_gz_search, a warp per chunk) and decodes from there without its window (k_gz_decode, a
// thread per chunk), into 16-bit symbols whose markers name bytes of the unknown 32 KB before the chunk.  The host then
// walks the chunks in order: chunk i must stop exactly where chunk i+1 started, or chunk i+1 guessed wrong and is
// decoded again from chunk i's end (the only sequential step, counted as "re-decoded").  k_gz_window carries the 32 KB
// windows from chunk to chunk, k_gz_resolve replaces every marker and narrows the symbols to bytes, k_gz_crc computes
// CRC-32 over pieces that the host combines in order.  Headers and trailers (a few bytes per member) are parsed on the
// host.  Memory depends on the chunk size (the span is kMaxChunks chunks), never on the file size.
#include "../../include/cfb200.h"
#include "cf_inflate.h"
#include "cf_buf.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

int cfb_fail_msg(int code, const char* msg);     // cfb200.cu: sets cfb_last_error()

namespace {

using cfz::NONE;
using cfz::WIN;

constexpr int kMaxChunks = 512;
constexpr uint32_t kCrcPiece = 32768;

struct ChunkIn { uint64_t start_bit, start_hdr, stop_bit; };

__global__ void __launch_bounds__(32) k_gz_search(const uint8_t* in, uint64_t n, const uint64_t* nominal, int n_chunks, uint64_t* found) {
	const int c = blockIdx.x + 1;
	if(c >= n_chunks) return;
	cfz::Tables t;
	const uint64_t lo = nominal[c], hi = c + 1 < n_chunks ? nominal[c + 1] : n * 8;
	uint64_t res = NONE;
	for(uint64_t base = lo; base < hi; base += 32) {
		const uint64_t p = base + threadIdx.x;
		const bool ok = p < hi && cfz::block_header_plausible(in, n, p, t);
		unsigned m = __ballot_sync(0xffffffffu, ok);
		while(m) {                        // the lowest plausible start decodes its whole block before it is taken
			const int l = __ffs(m) - 1;
			const bool good = __shfl_sync(0xffffffffu, (int)threadIdx.x == l && cfz::block_start_verified(in, n, p, t), l);
			if(good) { res = base + l; break; }
			m &= m - 1;
		}
		if(res != NONE) break;
	}
	if(threadIdx.x == 0) found[c] = res;
}

// one thread per block: the lanes of a warp would diverge on every symbol, so each chunk's decode gets a warp of its own
__global__ void __launch_bounds__(1) k_gz_decode(const uint8_t* in, uint64_t n, const ChunkIn* ci, int first, int count, uint16_t* sym, uint32_t cap,
                                                 cfz::ChunkResult* res) {
	const int i = blockIdx.x;
	if(i >= count) return;
	const int c = first + i;
	cfz::ChunkResult r;
	if(ci[c].start_bit == NONE) { memset(&r, 0, sizeof r); r.status = cfz::E_INPUT; r.end_bit = r.end_hdr = r.safe_bit = r.safe_hdr = NONE; res[c] = r; return; }
	cfz::Tables t;
	cfz::inflate_chunk(in, n, ci[c].start_bit, ci[c].start_hdr, ci[c].stop_bit, sym + (size_t)c * cap, cap, t, r);
	res[c] = r;
}

// win[0] = the window before chunk 0; win[c + 1] = the last 32 KB after chunk c (sequential over the chunks)
__global__ void k_gz_window(const uint16_t* sym, uint32_t cap, const uint32_t* n_sym, int k, uint8_t* win) {
	for(int c = 0; c < k; c++) {
		const uint16_t* s = sym + (size_t)c * cap; const uint64_t ns = n_sym[c];
		const uint8_t* pw = win + (size_t)c * WIN; uint8_t* nw = win + (size_t)(c + 1) * WIN;
		for(int j = threadIdx.x; j < WIN; j += blockDim.x) {
			const uint64_t v = ns + j;
			uint8_t x;
			if(v < (uint64_t)WIN) x = pw[v];
			else { const uint16_t y = s[v - WIN]; x = y < 256 ? (uint8_t)y : pw[(y - 256) & (WIN - 1)]; }
			nw[j] = x;
		}
		__syncthreads();
	}
}

// symbols of chunk blockIdx.y -> bytes at out + off[c]; a marker older than what the member has produced is an error
__global__ void k_gz_resolve(const uint16_t* sym, uint32_t cap, const uint32_t* n_sym, const uint64_t* off, const uint32_t* min_marker,
                             const uint8_t* win, uint8_t* out, int* err) {
	const int c = blockIdx.y;
	const uint16_t* s = sym + (size_t)c * cap; const uint8_t* w = win + (size_t)c * WIN; uint8_t* o = out + off[c];
	const uint32_t ns = n_sym[c], mm = min_marker[c];
	for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
		const uint16_t y = s[i];
		if(y < 256) { o[i] = (uint8_t)y; continue; }
		const uint32_t m = (y - 256u) & (WIN - 1);
		if(m < mm) atomicExch(err, 1);
		o[i] = w[m];
	}
}

// CRC-32 (reflected 0xEDB88320) of each kCrcPiece-byte piece of out[0, n)
__global__ void k_gz_crc(const uint8_t* out, uint64_t n, uint32_t* crc) {
	__shared__ uint32_t tab[256];
	for(int i = threadIdx.x; i < 256; i += blockDim.x) {
		uint32_t c = (uint32_t)i;
		for(int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1;
		tab[i] = c;
	}
	__syncthreads();
	const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, lo = p * kCrcPiece;
	if(lo >= n) return;
	const uint64_t hi = std::min<uint64_t>(n, lo + kCrcPiece);
	uint32_t c = 0xFFFFFFFFu;
	uint64_t i = lo;
	for(; i + 4 <= hi; i += 4) {
		const uint32_t w = *(const uint32_t*)(out + i);
		c = tab[(c ^ w) & 0xff] ^ (c >> 8);
		c = tab[(c ^ (w >> 8)) & 0xff] ^ (c >> 8);
		c = tab[(c ^ (w >> 16)) & 0xff] ^ (c >> 8);
		c = tab[(c ^ (w >> 24)) & 0xff] ^ (c >> 8);
	}
	for(; i < hi; i++) c = tab[(c ^ out[i]) & 0xff] ^ (c >> 8);
	crc[p] = c ^ 0xFFFFFFFFu;
}

// ---- CRC-32 algebra on the host (polynomials over GF(2), reflected), for combining piece CRCs in order
uint32_t multmodp(uint32_t a, uint32_t b) {
	uint32_t m = 1u << 31, p = 0;
	for(;;) {
		if(a & m) { p ^= b; if((a & (m - 1)) == 0) break; }
		m >>= 1;
		b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
	}
	return p;
}
uint32_t x2nmodp(uint64_t n, unsigned k) {      // x^(n * 2^k) mod p
	static uint32_t tab[32]; static bool init = false;
	if(!init) { uint32_t p = 1u << 30; tab[0] = p; for(int i = 1; i < 32; i++) tab[i] = p = multmodp(p, p); init = true; }
	uint32_t p = 1u << 31;
	while(n) { if(n & 1) p = multmodp(tab[k & 31], p); n >>= 1; k++; }
	return p;
}
uint32_t crc32_combine(uint32_t crc1, uint32_t crc2, uint64_t len2) { return multmodp(x2nmodp(len2, 3), crc1) ^ crc2; }
uint32_t crc32_host(uint32_t c, const uint8_t* p, size_t n) {       // member headers only (FHCRC)
	c = ~c;
	for(size_t i = 0; i < n; i++) { c ^= p[i]; for(int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1; }
	return ~c;
}

enum Phase { PH_HEADER = 0, PH_DEFLATE = 1, PH_TRAILER = 2 };

}  // namespace

struct cfb_gunzip {
	int device = 0; Stream st;
	uint64_t chunk = 64 << 10;      // compressed bytes per chunk
	uint32_t cap = 0;               // symbols per chunk
	DBuf<uint8_t> d_in, d_prev, d_win, d_out;      // d_prev: the window carried from the previous pass
	DBuf<uint16_t> d_sym; DBuf<ChunkIn> d_ci; DBuf<cfz::ChunkResult> d_res;
	DBuf<uint64_t> d_nom, d_found, d_off; DBuf<uint32_t> d_nsym, d_minm, d_crc; DBuf<int> d_err;
	HBuf<uint8_t> h_out; HBuf<uint32_t> h_crc;
	// stream state: bit offsets relative to the first byte the next call's input starts with
	int phase = PH_HEADER; uint64_t bit = 0, hdr = NONE;
	uint32_t crc = 0, win_len = 0; uint64_t msize = 0;
	uint64_t in_total = 0, out_total = 0, members = 0, chunks = 0, redone = 0;
	size_t pend_lo = 0, pend_hi = 0;
	int err = 0; std::string err_msg;
	~cfb_gunzip() { cudaSetDevice(device); if(st) cudaStreamSynchronize(st); }
};

namespace {

int gz_fail(cfb_gunzip* g, int code, const std::string& msg) {
	g->err = code; g->err_msg = msg;
	return cfb_fail_msg(code, msg.c_str());
}
#define GZ_CK(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) return gz_fail(g, CFB_ECUDA, std::string(#call " failed: ") + cudaGetErrorString(e_)); } while(0)

// RFC 1952 member header at p[0, n): 0 and *len when complete, 1 when more bytes are needed, < 0 on a bad header
int parse_header(cfb_gunzip* g, const uint8_t* p, uint64_t n, uint64_t* len) {
	if(n >= 1 && p[0] != 0x1f) return gz_fail(g, CFB_EDATA, "not in gzip format (trailing bytes after the last member?)");
	if(n >= 2 && p[1] != 0x8b) return gz_fail(g, CFB_EDATA, "not in gzip format (trailing bytes after the last member?)");
	if(n >= 3 && p[2] != 8) return gz_fail(g, CFB_EDATA, "unknown compression method");
	if(n >= 4 && (p[3] & 0xe0)) return gz_fail(g, CFB_EDATA, "reserved gzip header flags set");
	if(n < 10) return 1;
	const uint8_t flg = p[3];
	uint64_t q = 10;
	if(flg & 4) {                                       // FEXTRA
		if(n < q + 2) return 1;
		q += 2 + (uint64_t)(p[q] | (p[q + 1] << 8));
		if(n < q) return 1;
	}
	for(int f = 8; f <= 16; f <<= 1) if(flg & f) {     // FNAME, FCOMMENT: zero-terminated
		while(q < n && p[q]) q++;
		if(q >= n) return 1;
		q++;
	}
	if(flg & 2) {                                       // FHCRC: low 16 bits of the CRC-32 of the header so far
		if(n < q + 2) return 1;
		if((crc32_host(0, p, q) & 0xffff) != (uint32_t)(p[q] | (p[q + 1] << 8))) return gz_fail(g, CFB_EDATA, "header crc mismatch");
		q += 2;
	}
	*len = q;
	return 0;
}

inline int bit_at(const uint8_t* p, uint64_t n, uint64_t b) { return b < n * 8 ? (p[b >> 3] >> (b & 7)) & 1 : 0; }

// One pass of the DEFLATE stream from (g->bit, g->hdr) over in[0, n).  Output goes to h_out.
// *ended: the final block was decoded (g->bit = its end); otherwise g->bit/hdr hold the resume state.
int gz_pass(cfb_gunzip* g, const uint8_t* in0, uint64_t n0, bool is_last, bool* ended, uint64_t* produced) {
	*ended = false; *produced = 0;
	const uint64_t sb = std::min(g->bit, g->hdr) >> 3;           // first byte the decode reads
	const uint8_t* in = in0 + sb; const uint64_t n = n0 - std::min(sb, n0);
	const uint64_t bit = g->bit - sb * 8, hdr = g->hdr == NONE ? NONE : g->hdr - sb * 8;
	const uint64_t span = g->chunk * kMaxChunks;
	const uint64_t up = std::min<uint64_t>(n, 2 * span);
	const bool dev_last = is_last && up == n;
	if(up * 8 <= bit) {
		if(dev_last) return gz_fail(g, CFB_EDATA, cfz::status_text(cfz::E_INPUT));
		return 0;
	}
	const uint64_t avail_bits = up * 8 - bit, cb = g->chunk * 8;
	const uint64_t pass_stop = avail_bits > span * 8 ? bit + span * 8 : NONE;
	const int nch = (int)std::max<uint64_t>(1, std::min<uint64_t>(kMaxChunks, (std::min(avail_bits, span * 8) + cb - 1) / cb));
	std::vector<uint64_t> nom(nch + 1), found(nch, NONE);
	for(int c = 0; c < nch; c++) nom[c] = bit + (uint64_t)c * cb;
	nom[nch] = pass_stop;
	auto stop_of = [&](int c) { return c + 1 < nch ? nom[c + 1] : pass_stop; };
	GZ_CK(g->d_in.ensure_exact(up + 8)); GZ_CK(g->d_sym.ensure_exact((size_t)nch * g->cap)); GZ_CK(g->d_ci.ensure_exact(nch)); GZ_CK(g->d_res.ensure_exact(nch));
	GZ_CK(g->d_nom.ensure_exact(nch + 1)); GZ_CK(g->d_found.ensure_exact(nch)); GZ_CK(g->d_win.ensure_exact((size_t)(nch + 1) * WIN));
	GZ_CK(g->d_prev.ensure_exact(WIN));
	GZ_CK(cudaMemcpyAsync(g->d_win.p, g->d_prev.p, WIN, cudaMemcpyDeviceToDevice, g->st));
	GZ_CK(cudaMemcpyAsync(g->d_in.p, in, up, cudaMemcpyHostToDevice, g->st));
	if(nch > 1) {
		GZ_CK(cudaMemcpyAsync(g->d_nom.p, nom.data(), (nch + 1) * 8, cudaMemcpyHostToDevice, g->st));
		k_gz_search<<<nch - 1, 32, 0, g->st>>>(g->d_in.p, up, g->d_nom.p, nch, g->d_found.p);
		GZ_CK(cudaGetLastError());
		GZ_CK(cudaMemcpyAsync(found.data() + 1, g->d_found.p + 1, (nch - 1) * 8, cudaMemcpyDeviceToHost, g->st));
		GZ_CK(cudaStreamSynchronize(g->st));
	}
	std::vector<ChunkIn> ci(nch);
	ci[0] = ChunkIn{bit, hdr, stop_of(0)};
	for(int c = 1; c < nch; c++) ci[c] = ChunkIn{found[c], NONE, stop_of(c)};
	std::vector<cfz::ChunkResult> res(nch);
	GZ_CK(cudaMemcpyAsync(g->d_ci.p, ci.data(), nch * sizeof(ChunkIn), cudaMemcpyHostToDevice, g->st));
	k_gz_decode<<<nch, 1, 0, g->st>>>(g->d_in.p, up, g->d_ci.p, 0, nch, g->d_sym.p, g->cap, g->d_res.p);
	GZ_CK(cudaGetLastError());
	GZ_CK(cudaMemcpyAsync(res.data(), g->d_res.p, nch * sizeof(cfz::ChunkResult), cudaMemcpyDeviceToHost, g->st));
	GZ_CK(cudaStreamSynchronize(g->st));
	// walk the chunks in order: each one starts from a known state once the previous one is accepted
	std::vector<uint32_t> nsym;
	uint64_t end_bit = bit, end_hdr = hdr;
	for(int i = 0;; i++) {
		const cfz::ChunkResult& r = res[i];
		if(r.status < 0) {
			if(r.status == cfz::E_INPUT && !dev_last) { nsym.push_back(r.safe_sym); end_bit = r.safe_bit; end_hdr = r.safe_hdr; break; }
			return gz_fail(g, CFB_EDATA, cfz::status_text(r.status));
		}
		nsym.push_back(r.n_sym); end_bit = r.end_bit; end_hdr = r.end_hdr;
		if(r.status == cfz::ST_END) { *ended = true; break; }
		if(i + 1 == nch) break;
		const uint64_t f = found[i + 1];
		bool joins = r.end_hdr == NONE && f != NONE && r.end_bit == f;
		// a stored block decodes the same from any start whose three header bits and padding up to its byte are zero
		if(!joins && r.end_hdr == NONE && f != NONE && res[i + 1].first_type == 0 && r.end_bit < f && (r.end_bit + 10) / 8 == (f + 10) / 8) {
			joins = true;
			for(uint64_t b = r.end_bit; b < ((f + 10) / 8) * 8; b++) if(bit_at(in, up, b)) { joins = false; break; }
		}
		if(!joins) {
			const ChunkIn c1{r.end_bit, r.end_hdr, stop_of(i + 1)};
			found[i + 1] = r.end_bit;
			GZ_CK(cudaMemcpyAsync(g->d_ci.p + i + 1, &c1, sizeof c1, cudaMemcpyHostToDevice, g->st));
			k_gz_decode<<<1, 1, 0, g->st>>>(g->d_in.p, up, g->d_ci.p, i + 1, 1, g->d_sym.p, g->cap, g->d_res.p);
			GZ_CK(cudaGetLastError());
			GZ_CK(cudaMemcpyAsync(&res[i + 1], g->d_res.p + i + 1, sizeof(cfz::ChunkResult), cudaMemcpyDeviceToHost, g->st));
			GZ_CK(cudaStreamSynchronize(g->st));
			g->redone++;
		}
	}
	const int k = (int)nsym.size();
	g->chunks += nch;
	std::vector<uint64_t> off(k + 1, 0); std::vector<uint32_t> minm(k);
	uint64_t wl = g->win_len;
	for(int c = 0; c < k; c++) { off[c + 1] = off[c] + nsym[c]; minm[c] = (uint32_t)(WIN - wl); wl = std::min<uint64_t>(WIN, wl + nsym[c]); }
	const uint64_t total = off[k];
	if(total) {
		const uint64_t npieces = (total + kCrcPiece - 1) / kCrcPiece;
		GZ_CK(g->d_out.ensure_exact(total + 8)); GZ_CK(g->h_out.ensure_exact(total)); GZ_CK(g->d_crc.ensure_exact(npieces)); GZ_CK(g->h_crc.ensure_exact(npieces));
		GZ_CK(g->d_nsym.ensure_exact(k)); GZ_CK(g->d_minm.ensure_exact(k)); GZ_CK(g->d_off.ensure_exact(k + 1)); GZ_CK(g->d_err.ensure_exact(1));
		GZ_CK(cudaMemcpyAsync(g->d_nsym.p, nsym.data(), k * 4, cudaMemcpyHostToDevice, g->st));
		GZ_CK(cudaMemcpyAsync(g->d_minm.p, minm.data(), k * 4, cudaMemcpyHostToDevice, g->st));
		GZ_CK(cudaMemcpyAsync(g->d_off.p, off.data(), (k + 1) * 8, cudaMemcpyHostToDevice, g->st));
		GZ_CK(cudaMemsetAsync(g->d_err.p, 0, sizeof(int), g->st));
		k_gz_window<<<1, 1024, 0, g->st>>>(g->d_sym.p, g->cap, g->d_nsym.p, k, g->d_win.p);
		const uint32_t longest = *std::max_element(nsym.begin(), nsym.end());
		dim3 grid((unsigned)std::max<uint64_t>(1, std::min<uint64_t>(64, (longest + 4095) / 4096)), (unsigned)k);
		k_gz_resolve<<<grid, 256, 0, g->st>>>(g->d_sym.p, g->cap, g->d_nsym.p, g->d_off.p, g->d_minm.p, g->d_win.p, g->d_out.p, g->d_err.p);
		k_gz_crc<<<(unsigned)((npieces + 127) / 128), 128, 0, g->st>>>(g->d_out.p, total, g->d_crc.p);
		GZ_CK(cudaGetLastError());
		int derr = 0;
		GZ_CK(cudaMemcpyAsync(&derr, g->d_err.p, sizeof(int), cudaMemcpyDeviceToHost, g->st));
		GZ_CK(cudaMemcpyAsync(g->h_crc.p, g->d_crc.p, npieces * 4, cudaMemcpyDeviceToHost, g->st));
		GZ_CK(cudaMemcpyAsync(g->h_out.p, g->d_out.p, total, cudaMemcpyDeviceToHost, g->st));
		GZ_CK(cudaMemcpyAsync(g->d_prev.p, g->d_win.p + (size_t)k * WIN, WIN, cudaMemcpyDeviceToDevice, g->st));
		GZ_CK(cudaStreamSynchronize(g->st));
		if(derr) return gz_fail(g, CFB_EDATA, cfz::status_text(cfz::E_DIST));
		const uint32_t xp = x2nmodp(kCrcPiece, 3);
		uint32_t pc = 0;
		for(uint64_t p = 0; p + 1 < npieces; p++) pc = multmodp(xp, pc) ^ g->h_crc.p[p];
		const uint64_t last = total - (npieces - 1) * kCrcPiece;
		pc = npieces > 1 ? crc32_combine(pc, g->h_crc.p[npieces - 1], last) : g->h_crc.p[0];
		g->crc = crc32_combine(g->crc, pc, total);
		g->msize += total; g->win_len = (uint32_t)wl;
		g->pend_lo = 0; g->pend_hi = total;
	}
	g->out_total += total;
	*produced = total;
	g->bit = end_bit + sb * 8; g->hdr = end_hdr == NONE ? NONE : end_hdr + sb * 8;
	return 0;
}

}  // namespace

extern "C" int cfb_gunzip_create(int device, uint32_t chunk_kb, cfb_gunzip** out) {
	*out = NULL;
	int nd = 0;
	if(cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0) return cfb_fail_msg(CFB_ENODEV, "no CUDA device (the gzip inflater has no CPU fallback)");
	if(device < 0 || device >= nd) return cfb_fail_msg(CFB_EINVAL, "cfb_gunzip_create: no such device");
	if(chunk_kb == 0) { const char* e = getenv("CFB_GZ_CHUNK_KB"); chunk_kb = e ? (uint32_t)strtoul(e, NULL, 10) : 64; }
	if(chunk_kb < 1 || chunk_kb > 4096) return cfb_fail_msg(CFB_EINVAL, "gzip chunk size must be 1 to 4096 KB");
	if(cudaSetDevice(device) != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaSetDevice failed");
	std::unique_ptr<cfb_gunzip> g(new cfb_gunzip());
	g->device = device; g->chunk = (uint64_t)chunk_kb << 10;
	// FASTQ compresses 3-6x, and a chunk decodes one block past its end: a chunk that expands further than this stops
	// early and its successor is re-decoded, which serialises the pass
	g->cap = (uint32_t)(12 * g->chunk + 131072 + 258);
	if(g->st.create() != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaStreamCreate failed");
	*out = g.release();
	return CFB_OK;
}

extern "C" void cfb_gunzip_destroy(cfb_gunzip* g) { delete g; }

extern "C" int cfb_gunzip_run(cfb_gunzip* g, const void* in_, uint64_t n_in, int in_is_last, void* out, uint64_t out_cap,
                              uint64_t* n_out, uint64_t* n_consumed) {
	*n_out = 0; *n_consumed = 0;
	if(g->err) return cfb_fail_msg(g->err, g->err_msg.c_str());
	if(!in_ && n_in) return cfb_fail_msg(CFB_EINVAL, "cfb_gunzip_run: no input");
	if(cudaSetDevice(g->device) != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaSetDevice failed");
	const uint8_t* in = (const uint8_t*)in_;
	uint64_t pos = 0;
	bool passed = g->pend_hi > g->pend_lo;          // pending output is delivered before anything new is decoded
	for(;;) {
		if(g->phase == PH_HEADER) {
			if(pos == n_in) break;
			uint64_t len = 0;
			const int r = parse_header(g, in + pos, n_in - pos, &len);
			if(r < 0) return r;
			if(r == 1) { if(in_is_last) return gz_fail(g, CFB_EDATA, "truncated gzip header"); break; }
			pos += len;
			g->phase = PH_DEFLATE; g->bit = 0; g->hdr = NONE; g->crc = 0; g->msize = 0; g->win_len = 0;
		} else if(g->phase == PH_TRAILER) {
			if(n_in - pos < 8) { if(in_is_last) return gz_fail(g, CFB_EDATA, "truncated gzip trailer"); break; }
			const uint8_t* t = in + pos;
			const uint32_t crc = (uint32_t)t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
			const uint32_t isz = (uint32_t)t[4] | ((uint32_t)t[5] << 8) | ((uint32_t)t[6] << 16) | ((uint32_t)t[7] << 24);
			if(crc != g->crc) return gz_fail(g, CFB_EDATA, "crc-32 mismatch");
			if(isz != (uint32_t)g->msize) return gz_fail(g, CFB_EDATA, "length (ISIZE) mismatch");
			pos += 8; g->members++; g->phase = PH_HEADER;
		} else {
			if(passed) break;
			passed = true;
			bool ended = false; uint64_t produced = 0;
			const uint64_t b0 = g->bit, h0 = g->hdr;
			const int r = gz_pass(g, in + pos, n_in - pos, in_is_last != 0, &ended, &produced);
			if(r) return r;
			if(ended) { pos += (g->bit + 7) / 8; g->bit = 0; g->hdr = NONE; g->phase = PH_TRAILER; continue; }
			if(!produced && g->bit == b0 && g->hdr == h0) {
				if(n_in - pos > 2 * g->chunk * kMaxChunks) return gz_fail(g, CFB_EDATA, "deflate block larger than the inflater's span");
				break;                                  // needs more input
			}
			const uint64_t keep = std::min(g->bit, g->hdr) >> 3;
			pos += keep; g->bit -= keep * 8; if(g->hdr != NONE) g->hdr -= keep * 8;
		}
	}
	g->in_total += pos;
	*n_consumed = pos;
	const uint64_t give = std::min<uint64_t>(out_cap, g->pend_hi - g->pend_lo);
	if(give) { if(out) memcpy(out, g->h_out.p + g->pend_lo, give); g->pend_lo += give; }
	*n_out = give;
	return CFB_OK;
}

extern "C" int cfb_gunzip_get_state(const cfb_gunzip* g, cfb_gunzip_state* s) {
	if(g->err) return cfb_fail_msg(g->err, g->err_msg.c_str());
	if(g->pend_hi > g->pend_lo) return cfb_fail_msg(CFB_EINVAL, "cfb_gunzip_get_state: decompressed bytes are still pending");
	memset(s, 0, sizeof *s);
	s->in_offset = g->in_total; s->out_offset = g->out_total; s->bit = g->bit; s->hdr_bit = g->hdr; s->member_bytes = g->msize;
	s->crc = g->crc; s->win_len = g->win_len; s->phase = g->phase; s->members = (uint32_t)g->members;
	if(g->win_len) {
		if(cudaSetDevice(g->device) != cudaSuccess || cudaMemcpy(s->window, g->d_prev.p, WIN, cudaMemcpyDeviceToHost) != cudaSuccess)
			return cfb_fail_msg(CFB_ECUDA, "cfb_gunzip_get_state: window copy failed");
	}
	return CFB_OK;
}

extern "C" int cfb_gunzip_set_state(cfb_gunzip* g, const cfb_gunzip_state* s) {
	if(s->phase < PH_HEADER || s->phase > PH_TRAILER || s->win_len > (uint32_t)WIN || (s->phase != PH_DEFLATE && (s->bit || s->hdr_bit != NONE)))
		return cfb_fail_msg(CFB_EINVAL, "cfb_gunzip_set_state: invalid state");
	if(cudaSetDevice(g->device) != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaSetDevice failed");
	if(g->d_prev.ensure_exact(WIN) != cudaSuccess || cudaMemcpy(g->d_prev.p, s->window, WIN, cudaMemcpyHostToDevice) != cudaSuccess)
		return cfb_fail_msg(CFB_ECUDA, "cfb_gunzip_set_state: window copy failed");
	g->in_total = s->in_offset; g->out_total = s->out_offset; g->bit = s->bit; g->hdr = s->hdr_bit; g->msize = s->member_bytes;
	g->crc = s->crc; g->win_len = s->win_len; g->phase = s->phase; g->members = s->members;
	g->pend_lo = g->pend_hi = 0; g->err = 0; g->err_msg.clear();
	return CFB_OK;
}

extern "C" int cfb_gunzip_stats(const cfb_gunzip* g, uint64_t out[5]) {
	out[0] = g->members; out[1] = g->in_total; out[2] = g->out_total; out[3] = g->chunks; out[4] = g->redone;
	return CFB_OK;
}
