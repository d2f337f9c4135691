// cf_bunzip2.cu -- bzip2 decompressor on the device: the cfb_bunzip2_* entry points of include/cfb200.h.
//
// bzip2 blocks are independent (own tables, own MTF and run-length state, own CRC), so a pass over a span of compressed
// input decodes many blocks at once:
//   1. k_bz_scan tests every bit offset of the span for the 48-bit block and end-of-stream magics.
//   2. k_bz_decode decodes every block candidate (a thread per candidate, its tables and MTF list in shared memory)
//      into its BWT column L, its byte histogram and its end bit (cf_bzip2.h decode_block).
//   3. The host walks the chain from the known stream position: a block's end bit must be the next block magic or the
//      end-of-stream magic.  Candidates the chain skips are counted as rejected and their errors ignored.  A block that
//      does not start inside the span, or does not end inside the input, is left to the next pass.
//   4. The inverse BWT: k_bz_count / k_bz_cftab / k_bz_tt rank every byte of L among its equals (a warp per 4 KB
//      segment) and build tt[j] = (i << 8) | L[i] for the i-th byte sorted stably by value, then the LF walk from
//      tt[origPtr] is list-ranked: k_bz_rulers walks from every 128th node (and from the walk's first node) to the next
//      such ruler, k_bz_rank ranks the rulers on the walk's cycle, k_bz_walk walks again and writes.  A block whose
//      permutation has several cycles (a periodic block) repeats the first node's cycle, as libbz2's walk does.
//   5. RLE1: k_bz_rle_count runs every 4 KB segment of the walked bytes from each of the five possible run states,
//      k_bz_rle_chain picks each segment's true start state and output offset, k_bz_expand writes whole blocks into a
//      64 MB staging buffer with a CRC register per segment, and k_bz_crc combines them into the block CRC, which the
//      host checks together with the stream CRC.  A block expands at most 52x (46.6 MB): staging holds any block.
// Device memory depends on the blocks a pass holds (about 4.8 MB each, at most one per 128 KB of pass and 512 in all)
// and the staging buffer, never on the file size or on how far a block expands.
#include "../../include/cfb200.h"
#include "cf_bzip2.h"
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

using cbz::BLOCK_MAX;
using cbz::NONE;

constexpr uint32_t kSeg = 4096;                                  // bytes of L (and of the walked block) per segment
constexpr uint32_t kNSeg = (BLOCK_MAX + kSeg - 1) / kSeg;        // 220
constexpr uint32_t kRuler = 128;                                 // ruling-set stride of the LF walk
constexpr uint32_t kNR = (BLOCK_MAX + kRuler - 1) / kRuler + 1;  // regular rulers + the walk's first node
constexpr uint64_t kStage = 64ull << 20;                         // staging bytes: more than any block expands to
constexpr uint64_t kLook = 3ull << 20;                           // input past the span: more than any block's bits
static_assert(kLook * 8 >= cbz::MAX_BLOCK_BITS + 8, "a block the decoder accepts must fit in the look-ahead");
constexpr uint32_t kCandCap = 8192;
constexpr uint32_t kNoRank = 0xFFFFFFFFu;

struct BlkInfo { uint32_t slot, n, orig, nseg, cyc, total, err, pad; };

__global__ void __launch_bounds__(256) k_bz_scan(const uint8_t* in, uint64_t n, uint64_t lo, uint64_t hi, uint64_t* cand, uint32_t cap, uint32_t* count) {
	const uint64_t p0 = lo + ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 32;
	if(p0 >= hi) return;
	const uint64_t B = p0 >> 3;
	uint64_t h = 0, l = 0;
	for(int k = 0; k < 8; k++) { h = h << 8 | (B + k < n ? in[B + k] : 0); l = l << 8 | (B + 8 + k < n ? in[B + 8 + k] : 0); }
	const int sh = (int)(p0 & 7);
	for(int j = 0; j < 32; j++) {
		const int o = sh + j;
		const uint64_t v = (o ? (h << o) | (l >> (64 - o)) : h) >> 16;
		if(v != cbz::MAGIC_BLOCK && v != cbz::MAGIC_EOS) continue;
		const uint64_t p = p0 + j;
		if(p >= hi) break;
		const uint32_t k = atomicAdd(count, 1u);
		if(k < cap) cand[k] = p | (v == cbz::MAGIC_EOS ? 1ull << 63 : 0);
	}
}

// one thread per candidate block: a warp's lanes would diverge on every symbol
__global__ void __launch_bounds__(1) k_bz_decode(const uint8_t* in, uint64_t n, const uint64_t* bits, uint8_t* L, uint32_t* hist, cbz::BlockResult* res) {
	__shared__ cbz::Work w;
	const int i = blockIdx.x;
	cbz::BlockResult r;
	cbz::decode_block(in, n, bits[i], BLOCK_MAX, L + (size_t)i * BLOCK_MAX, w, r);
	res[i] = r;
	if(r.status == cbz::OK) for(int c = 0; c < 256; c++) hist[(size_t)i * 256 + c] = w.hist[c];
}

// byte counts of each segment of L: a warp per segment
__global__ void __launch_bounds__(256) k_bz_count(const uint8_t* L, const BlkInfo* blk, uint32_t* segcnt) {
	__shared__ uint32_t cnt[8][256];
	const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const BlkInfo bi = blk[blockIdx.y];
	const uint32_t seg = blockIdx.x * 8 + wp;
	if(seg >= bi.nseg) return;
	for(int c = lane; c < 256; c += 32) cnt[wp][c] = 0;
	__syncwarp();
	const uint8_t* l = L + (size_t)bi.slot * BLOCK_MAX;
	const uint32_t lo = seg * kSeg, hi = min(bi.n, lo + kSeg);
	for(uint32_t i = lo + lane; i < hi; i += 32) atomicAdd(&cnt[wp][l[i]], 1u);
	__syncwarp();
	uint32_t* o = segcnt + ((size_t)blockIdx.y * kNSeg + seg) * 256;
	for(int c = lane; c < 256; c += 32) o[c] = cnt[wp][c];
}

// segment counts -> each segment's first tt position per byte value (cftab + the counts of earlier segments)
__global__ void __launch_bounds__(256) k_bz_cftab(const uint32_t* hist, const BlkInfo* blk, uint32_t* segcnt) {
	__shared__ uint32_t h[256];
	const BlkInfo bi = blk[blockIdx.x];
	const int c = threadIdx.x;
	h[c] = hist[(size_t)bi.slot * 256 + c];
	__syncthreads();
	for(int d = 1; d < 256; d <<= 1) {              // inclusive scan
		const uint32_t v = c >= d ? h[c - d] : 0;
		__syncthreads();
		h[c] += v;
		__syncthreads();
	}
	uint32_t run = c ? h[c - 1] : 0;
	uint32_t* s = segcnt + (size_t)blockIdx.x * kNSeg * 256 + c;
	for(uint32_t g = 0; g < bi.nseg; g++) { const uint32_t v = s[(size_t)g * 256]; s[(size_t)g * 256] = run; run += v; }
}

// tt[cftab[L[i]]++] = (i << 8) | L[i], stable in i: a warp per segment, ranks among equal bytes by __match_any_sync
__global__ void __launch_bounds__(256) k_bz_tt(const uint8_t* L, const BlkInfo* blk, const uint32_t* segcnt, uint32_t* tt) {
	__shared__ uint32_t base[8][256];
	const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const BlkInfo bi = blk[blockIdx.y];
	const uint32_t seg = blockIdx.x * 8 + wp;
	if(seg >= bi.nseg) return;
	const uint32_t* s = segcnt + ((size_t)blockIdx.y * kNSeg + seg) * 256;
	for(int c = lane; c < 256; c += 32) base[wp][c] = s[c];
	__syncwarp();
	const uint8_t* l = L + (size_t)bi.slot * BLOCK_MAX;
	uint32_t* t = tt + (size_t)blockIdx.y * BLOCK_MAX;
	const uint32_t lo = seg * kSeg, hi = min(bi.n, lo + kSeg);
	const unsigned lt = (1u << lane) - 1;
	for(uint32_t i0 = lo; i0 < hi; i0 += 32) {
		const uint32_t i = i0 + lane;
		const bool ok = i < hi;
		const uint32_t c = ok ? l[i] : 256u + lane;
		const unsigned m = __match_any_sync(0xffffffffu, c);
		if(ok) {
			t[base[wp][c] + __popc(m & lt)] = i << 8 | c;
		}
		__syncwarp();
		if(ok && lane == 31 - __clz(m)) base[wp][c] += __popc(m);
		__syncwarp();
	}
}

__device__ __forceinline__ uint32_t first_node(const uint32_t* t, const BlkInfo& bi) { return t[bi.orig] >> 8; }
__device__ __forceinline__ uint32_t ruler_id(uint32_t q, uint32_t p0, uint32_t nreg) { return q % kRuler == 0 ? q / kRuler : (q == p0 ? nreg : kNoRank); }

// from every ruler, the number of LF steps to the next ruler and which it is
__global__ void __launch_bounds__(128) k_bz_rulers(const uint32_t* tt, const BlkInfo* blk, uint32_t* rnext, uint32_t* rdist) {
	const BlkInfo bi = blk[blockIdx.y];
	const uint32_t* t = tt + (size_t)blockIdx.y * BLOCK_MAX;
	const uint32_t nreg = (bi.n + kRuler - 1) / kRuler, p0 = first_node(t, bi);
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if(r > nreg || (r == nreg && p0 % kRuler == 0)) return;
	uint32_t q = r < nreg ? r * kRuler : p0, d = 0, id;
	do { q = t[q] >> 8; d++; id = ruler_id(q, p0, nreg); } while(id == kNoRank && d <= bi.n);
	rnext[(size_t)blockIdx.y * kNR + r] = id; rdist[(size_t)blockIdx.y * kNR + r] = d;
}

// the rulers on the first node's cycle, in walk order: their ranks and the cycle length (a thread per block)
__global__ void k_bz_rank(const uint32_t* tt, BlkInfo* blk, int nblk, const uint32_t* rnext, const uint32_t* rdist, uint32_t* rrank) {
	const int a = blockIdx.x * blockDim.x + threadIdx.x;
	if(a >= nblk) return;
	const BlkInfo bi = blk[a];
	const uint32_t nreg = (bi.n + kRuler - 1) / kRuler, p0 = first_node(tt + (size_t)a * BLOCK_MAX, bi);
	const uint32_t* nx = rnext + (size_t)a * kNR; const uint32_t* ds = rdist + (size_t)a * kNR; uint32_t* rk = rrank + (size_t)a * kNR;
	const uint32_t id0 = ruler_id(p0, p0, nreg);
	uint32_t r = id0, acc = 0;
	for(uint32_t guard = 0; guard <= nreg; guard++) {
		rk[r] = acc; acc += ds[r]; r = nx[r];
		if(r == id0 || r == kNoRank) break;
	}
	blk[a].cyc = acc;
	blk[a].err = r != id0;
}

// walk again from every ranked ruler and write its stretch of the block: byte k of the walk is D[k], k < n, repeating
// the cycle when it is shorter than the block.  D overwrites L, which tt already holds.
__global__ void __launch_bounds__(128) k_bz_walk(const uint32_t* tt, const BlkInfo* blk, const uint32_t* rdist, const uint32_t* rrank, uint8_t* L) {
	const BlkInfo bi = blk[blockIdx.y];
	const uint32_t* t = tt + (size_t)blockIdx.y * BLOCK_MAX;
	const uint32_t nreg = (bi.n + kRuler - 1) / kRuler;
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if(r > nreg || bi.err) return;
	const uint32_t R = rrank[(size_t)blockIdx.y * kNR + r];
	if(R == kNoRank) return;
	const uint32_t d = rdist[(size_t)blockIdx.y * kNR + r], c = bi.cyc, n = bi.n;
	uint8_t* D = L + (size_t)bi.slot * BLOCK_MAX;
	uint32_t q = r < nreg ? r * kRuler : first_node(t, bi);
	for(uint32_t j = 1; j <= d; j++) {
		const uint32_t e = t[q];
		q = e >> 8;
		uint32_t k = R + j;
		if(k >= c) k -= c;
		for(; k < n; k += c) D[k] = (uint8_t)e;
	}
}

// RLE1 of each segment from each start state 0..4: (end state, bytes out)
__global__ void __launch_bounds__(64) k_bz_rle_count(const uint8_t* L, const BlkInfo* blk, uint32_t* rlen, uint8_t* rend) {
	const BlkInfo bi = blk[blockIdx.y];
	const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
	if(seg >= bi.nseg) return;
	const uint8_t* D = L + (size_t)bi.slot * BLOCK_MAX;
	const uint32_t lo = seg * kSeg, hi = min(bi.n, lo + kSeg);
	int r[5] = {0, 1, 2, 3, 4}; uint32_t len[5] = {0, 0, 0, 0, 0};
	uint8_t prev = lo ? D[lo - 1] : 0;
	for(uint32_t i = lo; i < hi; i++) {
		const uint8_t x = D[i];
#pragma unroll
		for(int s = 0; s < 5; s++) len[s] += cbz::rle1_step(r[s], x, prev);
		prev = x;
	}
	const size_t o = ((size_t)blockIdx.y * kNSeg + seg) * 5;
	for(int s = 0; s < 5; s++) { rlen[o + s] = len[s]; rend[o + s] = (uint8_t)r[s]; }
}

// each segment's true start state and output offset; the block's output length (a thread per block)
__global__ void k_bz_rle_chain(BlkInfo* blk, int nblk, const uint32_t* rlen, const uint8_t* rend, uint8_t* seg_r, uint32_t* seg_off) {
	const int a = blockIdx.x * blockDim.x + threadIdx.x;
	if(a >= nblk) return;
	const BlkInfo bi = blk[a];
	int r = 0; uint32_t off = 0;
	for(uint32_t g = 0; g < bi.nseg; g++) {
		const size_t i = (size_t)a * kNSeg + g;
		seg_r[i] = (uint8_t)r; seg_off[i] = off;
		off += rlen[i * 5 + r]; r = rend[i * 5 + r];
	}
	blk[a].total = off;
	if(r == 4) blk[a].err = 2;
}

// expand every segment of the window's blocks into out at woff[block] + seg_off, with its CRC register from 0
__global__ void __launch_bounds__(64) k_bz_expand(const uint8_t* L, const BlkInfo* blk, const uint32_t* win, const uint64_t* woff,
                                                  const uint8_t* seg_r, const uint32_t* seg_off, uint8_t* out, uint32_t* seg_crc) {
	__shared__ uint32_t tab[256];
	for(int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = cbz::crc_table_entry(i);
	__syncthreads();
	const uint32_t a = win[blockIdx.y];
	const BlkInfo bi = blk[a];
	const uint32_t seg = blockIdx.x * blockDim.x + threadIdx.x;
	if(seg >= bi.nseg) return;
	const size_t si = (size_t)a * kNSeg + seg;
	const uint8_t* D = L + (size_t)bi.slot * BLOCK_MAX;
	const uint32_t lo = seg * kSeg, hi = min(bi.n, lo + kSeg);
	uint8_t* o = out + woff[blockIdx.y] + seg_off[si];
	int r = seg_r[si];
	uint8_t prev = lo ? D[lo - 1] : 0;
	uint32_t reg = 0;
	for(uint32_t i = lo; i < hi; i++) {
		const uint8_t x = D[i];
		if(r == 4) {
			for(uint32_t k = 0; k < x; k++) { *o++ = prev; reg = (reg << 8) ^ tab[(reg >> 24) ^ prev]; }
			r = 0;
		} else {
			r = r > 0 && x == prev ? r + 1 : 1;
			*o++ = x; reg = (reg << 8) ^ tab[(reg >> 24) ^ x];
		}
		prev = x;
	}
	seg_crc[si] = reg;
}

// block CRC = the segments' registers combined in order from the initial 0xFFFFFFFF (a thread per block)
__global__ void k_bz_crc(const BlkInfo* blk, const uint32_t* win, int nw, const uint32_t* seg_off, const uint32_t* seg_crc, uint32_t* bcrc) {
	const int y = blockIdx.x * blockDim.x + threadIdx.x;
	if(y >= nw) return;
	const uint32_t a = win[y];
	const BlkInfo bi = blk[a];
	uint32_t reg = 0xFFFFFFFFu;
	for(uint32_t g = 0; g < bi.nseg; g++) {
		const size_t i = (size_t)a * kNSeg + g;
		const uint32_t end = g + 1 < bi.nseg ? seg_off[i + 1] : bi.total;
		reg = cbz::crc_extend(reg, seg_crc[i], end - seg_off[i]);
	}
	bcrc[y] = ~reg;
}

enum Phase { PH_HEADER = 0, PH_BLOCKS = 1, PH_GARBAGE = 2 };
enum ItemKind { IT_BLOCK = 0, IT_EOS = 1 };
struct Item { int kind; uint32_t a; uint32_t crc; uint32_t total; };

}  // namespace

struct cfb_bunzip2 {
	int device = 0; Stream st;
	uint64_t span = 64ull << 20;    // compressed bytes scanned per pass
	uint32_t slots = 512;           // blocks decoded per pass
	DBuf<uint8_t> d_in, d_L, d_out, d_rend, d_segr; DBuf<uint64_t> d_cand, d_bits, d_woff;
	DBuf<uint32_t> d_count, d_hist, d_segcnt, d_tt, d_rnext, d_rdist, d_rrank, d_rlen, d_segoff, d_segcrc, d_win, d_bcrc;
	DBuf<cbz::BlockResult> d_res; DBuf<BlkInfo> d_blk;
	HBuf<uint8_t> h_out;            // pinned staging, kStage bytes
	// stream state: bit offset relative to the first byte the next call's input starts with
	int phase = PH_HEADER; uint64_t bit = 0; int level = 9; uint32_t scrc = 0; uint64_t headers = 0;
	std::vector<Item> items; size_t next_item = 0;      // the decoded pass, delivered in order
	uint64_t wait_for = 0;          // a block ran past the input: decode again once this many bytes are given
	uint64_t streams = 0, in_total = 0, out_total = 0, blocks = 0, rejected = 0, trailing = 0;
	size_t pend_lo = 0, pend_hi = 0;
	int err = 0; std::string err_msg;
	~cfb_bunzip2() { cudaSetDevice(device); if(st) cudaStreamSynchronize(st); }
};

namespace {

int bz_fail(cfb_bunzip2* g, int code, const std::string& msg) {
	g->err = code; g->err_msg = msg;
	return cfb_fail_msg(code, msg.c_str());
}
#define BZ_CK(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) return bz_fail(g, CFB_ECUDA, std::string(#call " failed: ") + cudaGetErrorString(e_)); } while(0)

uint32_t read32(const uint8_t* in, uint64_t n, uint64_t b) { cbz::Bits r; r.init(in, n, b); return r.peek(32); }

// Decode the blocks of one pass: scan, decode the candidates, chain them from the stream position (g->bit, g->phase)
// over in[0, n), then run the inverse BWT and the RLE1 counts of every accepted block.  Appends to g->items.
int bz_pass(cfb_bunzip2* g, const uint8_t* in0, uint64_t n0, bool is_last, bool* progress) {
	*progress = false;
	const uint64_t sb = g->bit >> 3;
	const uint8_t* in = in0 + sb; const uint64_t n = n0 - std::min(sb, n0);
	uint64_t b = g->bit - sb * 8;
	const uint64_t up = std::min<uint64_t>(n, g->span + kLook);
	const bool dev_last = is_last && up == n;
	// 1-2: candidates in [b, scan_hi), decoded in order up to the slot count
	std::vector<uint64_t> cands;
	std::vector<cbz::BlockResult> res;
	uint64_t scan_hi = std::min(up, g->span) * 8;
	if(scan_hi > b) {
		BZ_CK(g->d_in.ensure_exact(g->span + kLook + 16)); BZ_CK(g->d_cand.ensure_exact(kCandCap)); BZ_CK(g->d_count.ensure_exact(1));
		BZ_CK(cudaMemcpyAsync(g->d_in.p, in, up, cudaMemcpyHostToDevice, g->st));
		uint32_t count = 0;
		for(;;) {
			BZ_CK(cudaMemsetAsync(g->d_count.p, 0, 4, g->st));
			const uint64_t threads = (scan_hi - b + 31) / 32;
			k_bz_scan<<<(unsigned)((threads + 255) / 256), 256, 0, g->st>>>(g->d_in.p, up, b, scan_hi, g->d_cand.p, kCandCap, g->d_count.p);
			BZ_CK(cudaGetLastError());
			BZ_CK(cudaMemcpyAsync(&count, g->d_count.p, 4, cudaMemcpyDeviceToHost, g->st));
			BZ_CK(cudaStreamSynchronize(g->st));
			if(count <= kCandCap) break;
			scan_hi = b + std::max<uint64_t>(64, (scan_hi - b) / 4);          // too many candidates: scan less
		}
		std::vector<uint64_t> all(count);
		if(count) {
			BZ_CK(cudaMemcpyAsync(all.data(), g->d_cand.p, count * 8ull, cudaMemcpyDeviceToHost, g->st));
			BZ_CK(cudaStreamSynchronize(g->st));
		}
		for(uint64_t c : all) if(!(c >> 63)) cands.push_back(c);
		std::sort(cands.begin(), cands.end());
		const uint32_t k = (uint32_t)std::min<size_t>(cands.size(), g->slots);
		if(k) {
			res.resize(k);
			BZ_CK(g->d_bits.ensure_exact(k)); BZ_CK(g->d_L.ensure_exact((size_t)k * BLOCK_MAX)); BZ_CK(g->d_hist.ensure_exact((size_t)k * 256)); BZ_CK(g->d_res.ensure_exact(k));
			BZ_CK(cudaMemcpyAsync(g->d_bits.p, cands.data(), k * 8ull, cudaMemcpyHostToDevice, g->st));
			k_bz_decode<<<k, 1, 0, g->st>>>(g->d_in.p, up, g->d_bits.p, g->d_L.p, g->d_hist.p, g->d_res.p);
			BZ_CK(cudaGetLastError());
			BZ_CK(cudaMemcpyAsync(res.data(), g->d_res.p, k * sizeof(cbz::BlockResult), cudaMemcpyDeviceToHost, g->st));
			BZ_CK(cudaStreamSynchronize(g->st));
		}
	}
	// 3: the chain
	std::vector<BlkInfo> acc;
	size_t ci = 0;
	int ph = g->phase;
	const uint64_t b0 = b;
	for(;;) {
		if(ph == PH_HEADER) {                       // b is at a byte boundary
			const uint64_t B = b >> 3, avail = up > B ? up - B : 0;
			if(avail == 0) break;                   // more input, or the end of the file: the caller decides
			bool match = true;
			for(uint64_t i = 0; i < std::min<uint64_t>(avail, 4); i++)
				match = match && (i < 3 ? in[B + i] == (uint8_t)"BZh"[i] : in[B + 3] >= '1' && in[B + 3] <= '9');
			if(!match) {
				if(!g->headers) return bz_fail(g, CFB_EDATA, "not in bzip2 format");
				ph = PH_GARBAGE; *progress = true;  // bytes after a complete stream that are not a stream: ignored
				break;
			}
			if(avail < 4) { if(dev_last) return bz_fail(g, CFB_EDATA, "truncated bzip2 stream header"); break; }
			g->level = in[B + 3] - '0'; g->headers++;
			b += 32; ph = PH_BLOCKS; *progress = true;
			continue;
		}
		if(ph != PH_BLOCKS) break;
		if(b + 48 > up * 8) { if(dev_last) return bz_fail(g, CFB_EDATA, cbz::status_text(cbz::E_INPUT)); break; }
		const uint64_t m = cbz::read48(in, up, b);
		if(m == cbz::MAGIC_EOS) {
			if(b + 80 > up * 8) { if(dev_last) return bz_fail(g, CFB_EDATA, cbz::status_text(cbz::E_INPUT)); break; }
			g->items.push_back(Item{IT_EOS, 0, read32(in, up, b + 48), 0});
			b = (b + 80 + 7) & ~7ull; ph = PH_HEADER; *progress = true;
			continue;
		}
		if(m != cbz::MAGIC_BLOCK) return bz_fail(g, CFB_EDATA, cbz::status_text(cbz::E_MAGIC));
		while(ci < res.size() && cands[ci] < b) ci++;
		if(ci >= res.size() || cands[ci] != b) break;         // outside this pass's scan or slots: the next pass
		const cbz::BlockResult& r = res[ci];
		if(r.status == cbz::E_INPUT && !dev_last) {
			// the block ends in input not given yet, unless it already ran through more than any block can hold
			if(up - (b >> 3) >= kLook) return bz_fail(g, CFB_EDATA, "invalid block (longer than the format allows)");
			break;
		}
		if(r.status < 0) return bz_fail(g, CFB_EDATA, cbz::status_text(r.status));
		if(r.n > (uint32_t)g->level * 100000u) return bz_fail(g, CFB_EDATA, cbz::status_text(cbz::E_SIZE));
		g->items.push_back(Item{IT_BLOCK, (uint32_t)acc.size(), r.crc, 0});
		acc.push_back(BlkInfo{(uint32_t)ci, r.n, r.orig_ptr, (r.n + kSeg - 1) / kSeg, 0, 0, 0, 0});
		b = r.end_bit; ci++; *progress = true;
	}
	g->rejected += (uint64_t)(std::lower_bound(cands.begin(), cands.end(), b) - std::lower_bound(cands.begin(), cands.end(), b0)) - acc.size();
	g->bit = b + sb * 8; g->phase = ph;
	if(acc.empty()) return 0;
	// 4-5: inverse BWT and RLE1 counts of the accepted blocks
	const int na = (int)acc.size();
	BZ_CK(g->d_blk.ensure_exact(na)); BZ_CK(g->d_segcnt.ensure_exact((size_t)na * kNSeg * 256)); BZ_CK(g->d_tt.ensure_exact((size_t)na * BLOCK_MAX));
	BZ_CK(g->d_rnext.ensure_exact((size_t)na * kNR)); BZ_CK(g->d_rdist.ensure_exact((size_t)na * kNR)); BZ_CK(g->d_rrank.ensure_exact((size_t)na * kNR));
	BZ_CK(g->d_rlen.ensure_exact((size_t)na * kNSeg * 5)); BZ_CK(g->d_rend.ensure_exact((size_t)na * kNSeg * 5));
	BZ_CK(g->d_segr.ensure_exact((size_t)na * kNSeg)); BZ_CK(g->d_segoff.ensure_exact((size_t)na * kNSeg)); BZ_CK(g->d_segcrc.ensure_exact((size_t)na * kNSeg));
	BZ_CK(cudaMemcpyAsync(g->d_blk.p, acc.data(), na * sizeof(BlkInfo), cudaMemcpyHostToDevice, g->st));
	BZ_CK(cudaMemsetAsync(g->d_rrank.p, 0xff, (size_t)na * kNR * 4, g->st));
	const dim3 gseg((kNSeg + 7) / 8, na), grul((kNR + 127) / 128, na), grle((kNSeg + 63) / 64, na);
	const unsigned gb = (unsigned)((na + 31) / 32);
	k_bz_count<<<gseg, 256, 0, g->st>>>(g->d_L.p, g->d_blk.p, g->d_segcnt.p);
	k_bz_cftab<<<na, 256, 0, g->st>>>(g->d_hist.p, g->d_blk.p, g->d_segcnt.p);
	k_bz_tt<<<gseg, 256, 0, g->st>>>(g->d_L.p, g->d_blk.p, g->d_segcnt.p, g->d_tt.p);
	k_bz_rulers<<<grul, 128, 0, g->st>>>(g->d_tt.p, g->d_blk.p, g->d_rnext.p, g->d_rdist.p);
	k_bz_rank<<<gb, 32, 0, g->st>>>(g->d_tt.p, g->d_blk.p, na, g->d_rnext.p, g->d_rdist.p, g->d_rrank.p);
	k_bz_walk<<<grul, 128, 0, g->st>>>(g->d_tt.p, g->d_blk.p, g->d_rdist.p, g->d_rrank.p, g->d_L.p);
	k_bz_rle_count<<<grle, 64, 0, g->st>>>(g->d_L.p, g->d_blk.p, g->d_rlen.p, g->d_rend.p);
	k_bz_rle_chain<<<gb, 32, 0, g->st>>>(g->d_blk.p, na, g->d_rlen.p, g->d_rend.p, g->d_segr.p, g->d_segoff.p);
	BZ_CK(cudaGetLastError());
	BZ_CK(cudaMemcpyAsync(acc.data(), g->d_blk.p, na * sizeof(BlkInfo), cudaMemcpyDeviceToHost, g->st));
	BZ_CK(cudaStreamSynchronize(g->st));
	size_t j = 0;
	for(Item& it : g->items) if(it.kind == IT_BLOCK) {
		const BlkInfo& bi = acc[j++];
		if(bi.err == 1) return bz_fail(g, CFB_EDATA, "invalid BWT permutation");
		if(bi.err == 2) return bz_fail(g, CFB_EDATA, cbz::status_text(cbz::E_RLE));
		it.total = bi.total;
	}
	return 0;
}

// Deliver the next items of the decoded pass: expand whole blocks into staging, then check every block CRC and every
// stream CRC among them in order.  A window ends before the block that would overflow staging.
int bz_deliver(cfb_bunzip2* g) {
	std::vector<uint32_t> win; std::vector<uint64_t> off;
	uint64_t total = 0;
	size_t end = g->next_item;
	for(; end < g->items.size(); end++) {
		const Item& it = g->items[end];
		if(it.kind != IT_BLOCK) continue;
		if(total + it.total > kStage) break;
		win.push_back(it.a); off.push_back(total); total += it.total;
	}
	const int nw = (int)win.size();
	std::vector<uint32_t> got(nw);
	if(nw) {
		BZ_CK(g->d_out.ensure_exact(kStage)); BZ_CK(g->d_win.ensure_exact(nw)); BZ_CK(g->d_woff.ensure_exact(nw)); BZ_CK(g->d_bcrc.ensure_exact(nw));
		BZ_CK(g->h_out.ensure_exact(kStage));
		BZ_CK(cudaMemcpyAsync(g->d_win.p, win.data(), nw * 4ull, cudaMemcpyHostToDevice, g->st));
		BZ_CK(cudaMemcpyAsync(g->d_woff.p, off.data(), nw * 8ull, cudaMemcpyHostToDevice, g->st));
		k_bz_expand<<<dim3((kNSeg + 63) / 64, nw), 64, 0, g->st>>>(g->d_L.p, g->d_blk.p, g->d_win.p, g->d_woff.p, g->d_segr.p, g->d_segoff.p, g->d_out.p, g->d_segcrc.p);
		k_bz_crc<<<(nw + 31) / 32, 32, 0, g->st>>>(g->d_blk.p, g->d_win.p, nw, g->d_segoff.p, g->d_segcrc.p, g->d_bcrc.p);
		BZ_CK(cudaGetLastError());
		BZ_CK(cudaMemcpyAsync(got.data(), g->d_bcrc.p, nw * 4ull, cudaMemcpyDeviceToHost, g->st));
		BZ_CK(cudaMemcpyAsync(g->h_out.p, g->d_out.p, total, cudaMemcpyDeviceToHost, g->st));
		BZ_CK(cudaStreamSynchronize(g->st));
	}
	for(int i = 0; g->next_item < end; g->next_item++) {
		const Item& it = g->items[g->next_item];
		if(it.kind == IT_EOS) {
			if(it.crc != g->scrc) return bz_fail(g, CFB_EDATA, "stream CRC mismatch");
			g->scrc = 0; g->streams++;
			continue;
		}
		if(got[i] != it.crc) return bz_fail(g, CFB_EDATA, "block CRC mismatch");
		g->scrc = (g->scrc << 1 | g->scrc >> 31) ^ got[i];
		g->blocks++; i++;
	}
	g->out_total += total;
	g->pend_lo = 0; g->pend_hi = total;
	return 0;
}

}  // namespace

extern "C" int cfb_bunzip2_create(int device, uint32_t pass_kb, cfb_bunzip2** out) {
	*out = NULL;
	int nd = 0;
	if(cudaGetDeviceCount(&nd) != cudaSuccess || nd == 0) return cfb_fail_msg(CFB_ENODEV, "no CUDA device (the bzip2 decompressor has no CPU fallback)");
	if(device < 0 || device >= nd) return cfb_fail_msg(CFB_EINVAL, "cfb_bunzip2_create: no such device");
	if(pass_kb == 0) { const char* e = getenv("CFB_BZ2_PASS_KB"); pass_kb = e ? (uint32_t)strtoul(e, NULL, 10) : 65536; }
	if(pass_kb < 1 || pass_kb > (1u << 20)) return cfb_fail_msg(CFB_EINVAL, "bzip2 pass size must be 1 to 1048576 KB");
	if(cudaSetDevice(device) != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaSetDevice failed");
	std::unique_ptr<cfb_bunzip2> g(new cfb_bunzip2());
	g->device = device; g->span = (uint64_t)pass_kb << 10;
	// a level-9 block of FASTQ compresses to about 230 KB: a slot per 128 KB of span, at most 512 (about 2.5 GB)
	g->slots = (uint32_t)std::min<uint64_t>(512, std::max<uint64_t>(4, g->span >> 17));
	if(g->st.create() != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaStreamCreate failed");
	*out = g.release();
	return CFB_OK;
}

extern "C" void cfb_bunzip2_destroy(cfb_bunzip2* g) { delete g; }

extern "C" int cfb_bunzip2_run(cfb_bunzip2* g, const void* in_, uint64_t n_in, int in_is_last, void* out, uint64_t out_cap,
                               uint64_t* n_out, uint64_t* n_consumed) {
	*n_out = 0; *n_consumed = 0;
	if(g->err) return cfb_fail_msg(g->err, g->err_msg.c_str());
	if(!in_ && n_in) return cfb_fail_msg(CFB_EINVAL, "cfb_bunzip2_run: no input");
	if(cudaSetDevice(g->device) != cudaSuccess) return cfb_fail_msg(CFB_ECUDA, "cudaSetDevice failed");
	const uint8_t* in = (const uint8_t*)in_;
	uint64_t pos = 0;
	for(;;) {
		if(g->pend_hi > g->pend_lo) break;                // pending output is delivered before anything new is decoded
		if(g->next_item < g->items.size()) { const int r = bz_deliver(g); if(r) return r; continue; }
		g->items.clear(); g->next_item = 0;
		if(g->phase == PH_GARBAGE) { g->trailing += n_in - pos; pos = n_in; break; }
		if(!in_is_last && n_in - pos < g->wait_for) break;      // decoding the same block again would fail again
		bool progress = false;
		const int r = bz_pass(g, in + pos, n_in - pos, in_is_last != 0, &progress);
		if(r) return r;
		const uint64_t keep = std::min<uint64_t>(g->bit >> 3, n_in - pos);
		pos += keep; g->bit -= keep * 8;
		if(!progress) {
			if(g->phase == PH_BLOCKS && n_in - pos >= kLook) return bz_fail(g, CFB_EDATA, "invalid block (longer than the format allows)");
			// needs more input, or the file is complete.  Waiting for twice the input keeps the decodes of a block that
			// arrives in small pieces to a logarithmic number.
			g->wait_for = std::min<uint64_t>(2 * (n_in - pos), kLook);
			break;
		}
		g->wait_for = 0;
	}
	g->in_total += pos;
	*n_consumed = pos;
	const uint64_t give = std::min<uint64_t>(out_cap, g->pend_hi - g->pend_lo);
	if(give) { if(out) memcpy(out, g->h_out.p + g->pend_lo, give); g->pend_lo += give; }
	*n_out = give;
	return CFB_OK;
}

extern "C" int cfb_bunzip2_stats(const cfb_bunzip2* g, uint64_t out[6]) {
	out[0] = g->streams; out[1] = g->in_total; out[2] = g->out_total; out[3] = g->blocks; out[4] = g->rejected; out[5] = g->trailing;
	return CFB_OK;
}
