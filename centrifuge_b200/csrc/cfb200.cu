// cfb200.cu -- kernels + C ABI (include/cfb200.h) of the H100-native classification path.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo (see centrifuge_b200/build.py).
#include "../../include/cfb200.h"
#include "cf_index.h"
#include "cf_kernels.cuh"
#include "cf_buf.cuh"
#include "cf_nceil.h"
#include "cf_quals.h"
#include <cub/cub.cuh>

#include <algorithm>
#include <atomic>
#include <memory>
#include <mutex>
#include <thread>
#include <fcntl.h>
#include <unistd.h>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <set>
#include <string>
#include <vector>

using namespace cfb;

// =======================================================================================
// k_search
// =======================================================================================
enum { M_DONE = 0, M_FTAB = 1, M_LF = 2, M_NEED = 3, M_FTABK = 4, M_TASK = 5 };

struct SearchArgs {
	IndexView v; Params p; BatchView b;
	HitRec* hits; uint32_t* nhits; uint32_t cap;
	unsigned long long* task_ctr64; uint32_t ntasks, chunk;
	unsigned int* overflow;
	Counters* ctr;
	const uint64_t* pk; const uint32_t* nm; uint32_t W;   // packed reads (k_pack)
	uint32_t keep_short;                                  // store every hit (min_hitlen < 22, k_search_long); else only hits of >= kLongLen bases
};

__device__ __forceinline__ uint64_t shl64(uint64_t v, uint32_t n) {   // PTX shl clamps n >= 64 to "all shifted out"
	uint64_t r; asm("shl.b64 %0, %1, %2;" : "=l"(r) : "l"(v), "r"(n)); return r;
}
__device__ __forceinline__ uint64_t shr64(uint64_t v, uint32_t n) {
	uint64_t r; asm("shr.b64 %0, %1, %2;" : "=l"(r) : "l"(v), "r"(n)); return r;
}

// =======================================================================================
// k_pack: reads -> 2-bit words in *consumption order* of the backward search, both strands.
// Position p of a packed strand is the base the search looks at when dep == p:
//   strand 0 (fw): fw[rlen-1-p]      strand 1 (rc): comp(fw[p])      (Read::constructRevComps)
// base p sits in bits 2*(p&31) of word p>>5; N -> code 0 plus a bit in the parallel N mask.
// =======================================================================================
struct PackArgs { BatchView b; uint64_t* pk; uint32_t* nm; uint32_t W; };

// 4 bytes at an arbitrary byte offset of a 4-byte aligned buffer (reads at most 7 bytes past `off`: device
// buffers carry that much slack)
__device__ __forceinline__ uint32_t load4(const uint8_t* base, uint64_t off) {
	const uint32_t* w = reinterpret_cast<const uint32_t*>(base + (off & ~3ull));
	return __funnelshift_r(w[0], w[1], (uint32_t)(off & 3) * 8);
}

// four 2-bit fields held one per byte -> 8 contiguous bits; four 1-bit flags held one per byte -> 4 bits
__device__ __forceinline__ uint32_t squeeze4x2(uint32_t x) { x = (x | (x >> 6)) & 0x000F000Fu; return (x | (x >> 12)) & 0xFFu; }
__device__ __forceinline__ uint32_t squeeze4x1(uint32_t x) { x = (x | (x >> 7)) & 0x00030003u; return (x | (x >> 14)) & 0xFu; }

__global__ void __launch_bounds__(128) k_pack(const PackArgs a) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;      // (task, word)
	const uint64_t ntasks = (uint64_t)a.b.n_units * a.b.n_mates * 2;
	if(i >= ntasks * a.W) return;
	const uint64_t t = i / a.W; const uint32_t k = (uint32_t)(i - t * a.W);
	const uint32_t per = 2u * (uint32_t)a.b.n_mates;
	const uint32_t unit = (uint32_t)(t / per), rem = (uint32_t)(t - (uint64_t)unit * per);
	const int mate = (int)(rem >> 1), strand = (int)(rem & 1);
	const uint32_t len = mate ? a.b.len[1][unit] : a.b.len[0][unit];        // no runtime index into the parameter arrays
	uint64_t w = 0; uint32_t n = 0;
	if(k * 32 < len) {
		const uint64_t off = mate ? a.b.off[1][unit] : a.b.off[0][unit];
		const uint32_t cnt = min(32u, len - k * 32);         // bases of this word
		// strand 1 consumes fw[p], strand 0 consumes fw[len-1-p]: either way a window of `cnt` consecutive bytes,
		// packed in window order four bytes at a time and flipped end to end for strand 0
		const uint64_t lo = strand ? off + k * 32 : off + (len - k * 32 - cnt);
		#pragma unroll
		for(uint32_t g = 0; g < 32; g += 4) {
			if(g < cnt) {
				const uint32_t keep = cnt - g >= 4 ? 0xffffffffu : ((1u << (8 * (cnt - g))) - 1u);
				const uint32_t v = load4(a.b.bases, lo + g) & keep;
				const uint32_t nb = __vcmpne4(v & 0xFCFCFCFCu, 0u) & 0x01010101u;        // codes above 3 are N
				uint32_t b2 = v & 0x03030303u;
				if(strand) b2 ^= 0x03030303u & keep;
				b2 &= ~(nb * 3u);
				w |= (uint64_t)squeeze4x2(b2) << (2 * g);
				n |= squeeze4x1(nb) << g;
			}
		}
		if(!strand) {
			uint64_t x = __brevll(w);
			x = ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);
			w = x >> (2 * (32 - cnt)); n = __brev(n) >> (32 - cnt);
		}
	}
	a.pk[i] = w; a.nm[i] = n;
}

// ---------------------------------------------------------------------------------------
// Work distribution for the thread-per-walk kernels: a warp owns a pool [base, end) of task ids
// refilled with ONE global atomic per `chunk` (>= 32) tasks; lanes that need work take consecutive
// ids by ballot rank at a convergent point of the loop.  (A per-lane atomicAdd on one address
// serialises in L2: ~1M same-address atomics cost more than the whole resolve kernel.)  pool_ahead issues the
// atomic of the next refill as soon as the pool cannot serve a full warp any more and leaves its result in the pool, so
// that the refill itself waits for nothing.
// ---------------------------------------------------------------------------------------
struct WarpPool { unsigned long long base = 0, end = 0, next = 0; bool ahead = false; };      // ahead: lane 0's `next` is the next chunk
__device__ __forceinline__ void pool_ahead(WarpPool& P, unsigned long long* ctr, unsigned chunk) {
	if(!P.ahead && P.end - P.base < 32) { if((threadIdx.x & 31) == 0) P.next = atomicAdd(ctr, (unsigned long long)chunk); P.ahead = true; }
}
__device__ __forceinline__ bool pool_take(WarpPool& P, bool want, unsigned long long* ctr, unsigned long long total, unsigned chunk, unsigned long long& out) {
	const unsigned need = __ballot_sync(0xffffffffu, want);
	if(!need) return false;
	const unsigned lane = threadIdx.x & 31;
	const unsigned cnt = __popc(need), r = __popc(need & ((1u << lane) - 1u));
	const unsigned long long avail = P.end - P.base;
	unsigned long long nb = 0;
	const bool refill = avail < cnt;
	if(refill) { if(lane == 0) nb = P.ahead ? P.next : atomicAdd(ctr, (unsigned long long)chunk); nb = __shfl_sync(0xffffffffu, nb, 0); P.ahead = false; }
	unsigned long long t, lim;
	if(r < avail) { t = P.base + r; lim = P.end; }
	else { t = nb + (r - avail); lim = nb + chunk < total ? nb + chunk : total; }
	if(refill) { P.base = nb + (cnt - avail); P.end = nb + chunk < total ? nb + chunk : total; if(P.base > P.end) P.base = P.end; }
	else P.base += cnt;
	out = t;
	return want && t < lim;
}

__device__ __forceinline__ uint64_t even_bits(uint64_t x) {    // gather bits 0,2,4,.. into the low 32 bits
	x &= 0x5555555555555555ull;
	x = (x | (x >> 1)) & 0x3333333333333333ull;
	x = (x | (x >> 2)) & 0x0f0f0f0f0f0f0f0full;
	x = (x | (x >> 4)) & 0x00ff00ff00ff00ffull;
	x = (x | (x >> 8)) & 0x0000ffff0000ffffull;
	x = (x | (x >> 16)) & 0x00000000ffffffffull;
	return x;
}

// ---------------------------------------------------------------------------------------
// rank16 (format: cf_logic.h, r16_entry / r16_lf): the layout both walk kernels use.  LF(row, c) costs ONE 16-byte load request.
// Measured on this part (tools/gather_bench.cu): fully divergent gathers are capped at ~70 G 16-byte
// lane requests/s independent of size (32 B: 34 G/s, 64 B: 17.6 G/s, 128 B: 8.9 G/s), so requests per
// LF step -- not bytes -- is what bounds the walk.  The four bases of a block share one 64-byte chunk.
// ---------------------------------------------------------------------------------------
__global__ void k_build_rank16(const uint64_t* sides, uint64_t num_sides, uint64_t zside, uint32_t zoffc, uint64_t* r16) {
	const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(b > num_sides * 6) return;
	const bool sentinel = b == num_sides * 6;                 // totals, for an exclusive bound == len+1 on a side boundary
	const uint64_t s = sentinel ? num_sides - 1 : b / 6; const uint32_t sub = sentinel ? 6u : (uint32_t)(b - s * 6);
	const uint64_t* sd = sides + s * 16;
	uint64_t occ[4] = {sd[12], sd[13], sd[14], sd[15]};
	for(uint32_t k = 0; k < sub * 2; k++) {
		const uint64_t w = sd[k];
		const uint64_t lo = w & 0x5555555555555555ull, hi = (w >> 1) & 0x5555555555555555ull;
		const uint32_t c1 = __popcll(lo & ~hi), c2 = __popcll(hi & ~lo), c3 = __popcll(hi & lo);
		occ[1] += c1; occ[2] += c2; occ[3] += c3; occ[0] += 32 - c1 - c2 - c3;
	}
	if(s == zside && zoffc < sub * 64) occ[0] -= 1;
	for(int c = 0; c < 4; c++) {
		uint64_t bits = 0;
		if(!sentinel) {
			bits = even_bits(match2(sd[sub * 2], c)) | (even_bits(match2(sd[sub * 2 + 1], c)) << 32);
			if(c == 0 && s == zside && zoffc >= sub * 64 && zoffc < sub * 64 + 64) bits &= ~(1ull << (zoffc - sub * 64));
		}
		r16[(b * 4 + c) * 2] = occ[c]; r16[(b * 4 + c) * 2 + 1] = bits;
	}
}
__global__ void k_mark_boundaries(const uint64_t* brow, uint32_t n, uint64_t* r16) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) atomicOr((unsigned long long*)&r16[(brow[i] >> 6) * 8], 1ull << 63);
}
// compact rank layout (format: cf_logic.h, cr_convert_side / cr_lf): the superblock table first, from the file's sides, then
// one thread per side converts it in place
__global__ void k_cr_superblocks(const uint64_t* sides, uint64_t num_sides, uint64_t zoff, uint64_t nsb, uint64_t* sb) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < nsb) cr_sb_entry(sides, num_sides, zoff, i, sb + i * 4);
}
__global__ void k_cr_convert(uint64_t* sides, uint64_t num_sides, uint64_t zoff, const uint64_t* sb) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < num_sides) cr_convert_side(sides, num_sides, zoff, sb, i);
}
__global__ void k_build_ftab2(IndexView v, uint64_t n, uint64_t* ftab2) {
	const uint64_t fi = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(fi >= n) return;
	ftab2[fi * 2] = ftab_hi(v, v.ftab[fi]); ftab2[fi * 2 + 1] = ftab_lo(v, v.ftab[fi + 1]);
}
// The nhits[] word of a strand list (nh_pack), which hits k_search_t stores, and the rules by which k_prep restores what it
// left out (list_dropped, list_needs_regen, list_needs_exact_ranges): cf_logic.h, where the CPU tests compile them too.  k_prep
// regenerates a list with a one-thread version of the kernel's walk (search_strand_dev); storing only the long hits removes
// most of the hit traffic (random partial-sector writes) and shrinks the per-read device footprint from ~3.6 KB to ~2.3 KB.

// K-mer jump table: one 16-byte entry per K-mer (K >= ftabChars) that a partial search gathers in place of its first K
// steps (hi_aligner.h:985-1008), trading HBM capacity (16 B x 4^K; 17 GB at K = 15) for random accesses.
//   x = top | (bot - top) << 40: the SA range partialSearch reaches after K bases, obtained by K - ftabChars LF steps from
//       the 10-mer range.  A width of 0 says the range died somewhere in between, kFtabkWide that it is too wide to store;
//       either way the kernel redoes that search from the 10-mer table.  Rows need 40 bits (tables are built below 2^40 rows).
//   y = death bitmap: bit e is set when the (K+3)-mer of extension e = c_K | c_{K+1} << 2 | c_{K+2} << 4 occurs.  A partial
//       search on a strand that does not match -- most searches of most reads -- dies within these three bases, and the
//       bitmap gives the length of the hit partialSearch would report (ftabk_death), so the search costs this ONE gather
//       instead of one or two rank gathers per base after it.  Its SA range is not computed, which is fine because a hit
//       shorter than min_hitlen is never resolved (k_prep recomputes the range in the rare cases where a short hit's size can
//       influence the result).  All ones = always continue from the range: for absent K-mers, when the bitmap is not wanted,
//       and where the decode would be wrong (near the text start a (K+1)- or (K+2)-mer can occur with none of its 3-extensions).
static const uint64_t kFtabkWide = 0xFFFFFFull;
// 0 = the search goes on from the stored range; 1, 2, 3 = the range dies after K, K+1, K+2 bases (a hit of K + v - 1 bases)
__device__ __forceinline__ uint32_t ftabk_death(uint64_t y, uint32_t e) {
	if((y >> e) & 1ull) return 0;
	if(!(y & (0x1111111111111111ull << (e & 3u)))) return 1;      // no occurring extension starts with c_K
	if(!(y & (0x0001000100010001ull << (e & 15u)))) return 2;     // none starts with c_K c_{K+1}
	return 3;
}
// One thread per K-mer walks the depth-3 tree of extensions; a 64-byte rank16 chunk carries the entries of all four bases of
// a block, so every tree node costs one or two loads.  On the compact rank layout the walk takes cr_lf instead.
__device__ __forceinline__ void lf4(const IndexView& v, const ulonglong2* r16, uint64_t top, uint64_t bot, uint64_t t[4], uint64_t b[4]) {
	if(v.cr) { for(int c = 0; c < 4; c++) { t[c] = cr_lf(v, top, c); b[c] = cr_lf(v, bot, c); } return; }
	const ulonglong2* pt = r16 + r16_entry(top, 0); const ulonglong2* pb = r16 + r16_entry(bot, 0);
	#pragma unroll
	for(int c = 0; c < 4; c++) {
		const ulonglong2 et = __ldg(pt + c); const ulonglong2 eb = (pb == pt) ? et : __ldg(pb + c);
		t[c] = r16_lf(v, top, c, et.x, et.y);
		b[c] = r16_lf(v, bot, c, eb.x, eb.y);
	}
}
__global__ void __launch_bounds__(128) k_build_ftabk(IndexView v, int K, uint64_t n, bool death, ulonglong2* out) {
	const uint64_t fk = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(fk >= n) return;
	const ulonglong2* r16 = reinterpret_cast<const ulonglong2*>(v.rank16);
	const int fc = v.ftab_chars;
	const uint64_t f10 = fk & ((1ull << (2 * fc)) - 1ull);
	uint64_t top = v.ftab2[f10 * 2], bot = v.ftab2[f10 * 2 + 1];
	for(int j = fc; j < K && bot > top; j++) {
		const int c = (int)((fk >> (2 * j)) & 3);
		if(v.cr) { top = cr_lf(v, top, c); bot = cr_lf(v, bot, c); continue; }
		const ulonglong2 tq = __ldg(r16 + r16_entry(top, c)), bq = __ldg(r16 + r16_entry(bot, c));
		top = r16_lf(v, top, c, tq.x, tq.y);
		bot = r16_lf(v, bot, c, bq.x, bq.y);
	}
	if(bot <= top) { out[fk] = make_ulonglong2(0ull, ~0ull); return; }
	uint64_t y = ~0ull;
	if(death) {
		// true death depth of every extension (0 = the (K+3)-mer occurs), then the bitmap, kept only if it decodes to them all
		uint8_t dv[64];
		uint64_t t1[4], b1[4]; lf4(v, r16, top, bot, t1, b1);
		for(int c0 = 0; c0 < 4; c0++) {
			if(b1[c0] <= t1[c0]) { for(int r = 0; r < 16; r++) dv[c0 | (r << 2)] = 1; continue; }
			uint64_t t2[4], b2[4]; lf4(v, r16, t1[c0], b1[c0], t2, b2);
			for(int c1 = 0; c1 < 4; c1++) {
				if(b2[c1] <= t2[c1]) { for(int c2 = 0; c2 < 4; c2++) dv[c0 | (c1 << 2) | (c2 << 4)] = 2; continue; }
				uint64_t t3[4], b3[4]; lf4(v, r16, t2[c1], b2[c1], t3, b3);
				for(int c2 = 0; c2 < 4; c2++) dv[c0 | (c1 << 2) | (c2 << 4)] = b3[c2] <= t3[c2] ? 3 : 0;
			}
		}
		y = 0;
		for(int e = 0; e < 64; e++) if(dv[e] == 0) y |= 1ull << e;
		for(uint32_t e = 0; e < 64; e++) if(ftabk_death(y, e) != dv[e]) { y = ~0ull; break; }
	}
	const uint64_t w = bot - top;
	out[fk] = make_ulonglong2(top | ((w < kFtabkWide ? w : kFtabkWide) << 40), y);
}

// ---------------------------------------------------------------------------------------
// k_search_t: one thread per walk.  No cross-lane traffic: each lane reads the 32-byte rank sectors of
// its own top and bot rows.  The packed strand of the current task lives in registers (RW words, reads
// up to 32*RW bases), so the per-step base, the N test and the 10-mer ftab index are register extracts.
// A loop trip has three parts:
//   fetch    every lane issues the one or two 16-byte gathers its walk needs, whatever table it is at; a lane that took a
//            task in the previous trip (M_TASK) issues the loads of its read instead: flags, length, packed strand.  These
//            are the only loads of the trip whose result the trip waits for, and they are all in flight together.
//   consume  a branch per table.  A branch only computes: it advances top / bot / dep, or says that the partial search
//            ended and leaves the hit in registers.  The 32 walks of a warp are independent, so most trips run most branches.
//   restart  the ONE copy of the hit store, the restart policy and the next partial search's prologue, run once per trip by
//            all lanes whose search ended or whose read arrived.  (Inlined at each of the eight places a search can end, it was
//            nine tenths of the loop's instructions, and a warp ran most copies one after the other in every trip.)
// One loop trip = one DRAM round trip for every walk of the warp.
// ---------------------------------------------------------------------------------------
template <int RW> struct ReadRegs {
	uint64_t rw[RW]; uint32_t nw[RW];
	__device__ __forceinline__ uint64_t word(uint32_t k) const {
		uint64_t v = 0;
		#pragma unroll
		for(int q = 0; q < RW; q++) if((uint32_t)q == k) v = rw[q];
		return v;
	}
	__device__ __forceinline__ uint32_t nword(uint32_t k) const {
		uint32_t v = 0;
		#pragma unroll
		for(int q = 0; q < RW; q++) if((uint32_t)q == k) v = nw[q];
		return v;
	}
	// base at search depth p (4 = N)
	__device__ __forceinline__ int base(uint32_t p) const {
		const uint32_t k = p >> 5, sh = p & 31;
		return ((nword(k) >> sh) & 1u) ? 4 : (int)((word(k) >> (2 * sh)) & 3);
	}
	// bases p .. p+31 (base p in the low bits) and their N bits
	__device__ __forceinline__ void window(uint32_t p, uint64_t& win, uint32_t& nwin) const {
		const uint32_t k = p >> 5, sh = p & 31;
		win = shr64(word(k), 2 * sh) | shl64(word(k + 1), 64 - 2 * sh);
		nwin = (uint32_t)(((uint64_t)nword(k) | ((uint64_t)nword(k + 1) << 32)) >> sh);
	}
};

// Loads of the fetch point: predicated, and volatile asm so that the compiler can neither sink a load into the branch that
// consumes it nor hoist a consumer's wait above the other loads.  A lane whose predicate is off keeps the register's value.
__device__ __forceinline__ void ld_if(ulonglong2& v, const void* p) {      // on = p is not null
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u64 p, %2, 0;\n\t@p ld.global.nc.v2.u64 {%0, %1}, [%2];\n\t}" : "+l"(v.x), "+l"(v.y) : "l"(p));
}
__device__ __forceinline__ void ld_if(uint64_t& v, const uint64_t* p, bool on) {
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u64 %0, [%1];\n\t}" : "+l"(v) : "l"(p), "r"((uint32_t)on));
}
__device__ __forceinline__ void ld_if(uint32_t& v, const uint32_t* p, bool on) {
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u32 %0, [%1];\n\t}" : "+r"(v) : "l"(p), "r"((uint32_t)on));
}
__device__ __forceinline__ void ld_if(uint32_t& v, const uint8_t* p, bool on) {
	asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u8 %0, [%1];\n\t}" : "+r"(v) : "l"(p), "r"((uint32_t)on));
}

// REQS: count the product's own load requests with every table live (what the roofline of *this* kernel is made of), and how
// the loop spends its trips (Counters::it_*, clk_*).  The reference's operation counters come from search_strand_scalar
// (k_search_long<true>).
template <bool REQS, int RW>
__global__ void __launch_bounds__(kSearchThreads, !REQS && RW <= 5 ? 8 : 1) k_search_t(const SearchArgs a) {
	// RW = 4: 62 registers, RW = 5: 64 under the launch bounds, neither spills: 8 CTAs per SM.  A ninth CTA needs 56.  The random-gather
	// probe reaches its ceiling with these 1024 walks in flight per SM (tools/search_iter_stats.py), so the walks in flight are not
	// the limit; what a trip spends outside its one wait for memory is (DESIGN.md 4, 6)
	const ulonglong2* r16 = reinterpret_cast<const ulonglong2*>(a.v.rank16);
	const ulonglong2* ftab2 = reinterpret_cast<const ulonglong2*>(a.v.ftab2);
	const ulonglong2* ftabk = reinterpret_cast<const ulonglong2*>(a.v.ftabk);
	const uint32_t fk = a.v.ftabk ? (uint32_t)a.v.ftabk_chars : 0u;
	const uint32_t fc = (uint32_t)a.v.ftab_chars;
	const unsigned long long* w8 = reinterpret_cast<const unsigned long long*>(a.v.walk8);
	// death bitmap of the K-mer table (fd = K + 3): only while every hit it can end (at most fd - 1 bases) stays below
	// min_hitlen, i.e. is never resolved
	const uint32_t fd = (fk == 0 || a.p.min_hitlen < (uint32_t)a.v.ftabd_chars) ? 0u : (uint32_t)a.v.ftabd_chars;
	const uint32_t msh = a.b.n_mates == 2 ? 2u : 1u;      // task = (unit << msh) | mate << 1 | strand
	ReadRegs<RW> rd;
	#pragma unroll
	for(int k = 0; k < RW; k++) { rd.rw[k] = 0; rd.nw[k] = 0; }
	uint64_t top = 0, bot = 0, fi = 0;      // M_FTABK: fi = K-mer | (64 | extension) << 2K when the bitmap applies
	uint32_t rlen = 0, tid = 0, cur = 0, dep = 0, offset = 0, nh = 0, nt = 0, slow_until = 0, fail_at = 0xffffffffu;
	bool nolong = true;      // no hit of this strand reaches min_hitlen (kListNoLong tells the per-unit kernels)
	int mode = M_NEED;
	unsigned long long q_r16 = 0, q_f2 = 0, q_fk = 0, q_w8 = 0;
	unsigned long long q_w1 = 0, q_w24 = 0, q_w5 = 0, j_row = 0, j_row_ok = 0, j_rng = 0, j_rng_ok = 0, j_w5_ok = 0;
	// REQS: trip statistics.  paths = consumer branches (bits 0-15) and restart blocks (bits 16-) this lane ran in this trip
	unsigned long long s_trips = 0, s_lreq = 0, s_cons = 0, s_rest = 0, s_task = 0, s_head = 0, s_wait = 0, s_tail = 0;
	uint32_t paths = 0; long long t_top = 0, t_issue = 0, t_data = 0;
	WarpPool pool;
	bool more = true;      // warp-uniform: the global task counter is not exhausted yet

	for(;;) {
		// ---------------- hand out tasks (convergent point) ----------------
		// A lane only takes the task's number here.  Its read is loaded at the fetch point below with everybody's gathers and
		// its first search starts in this trip's restart block, so no load is waited for on its own.
		if(REQS) { paths = 0; t_top = clock64(); }
		{
			const bool want = mode == M_NEED;
			if(more) {
				unsigned long long t = 0;
				const bool got = pool_take(pool, want, a.task_ctr64, (unsigned long long)a.ntasks, a.chunk, t);
				if(want) {
					if(got) { tid = (uint32_t)t; mode = M_TASK; if(REQS) paths |= 1u << 17; }
					else mode = M_DONE;
				}
				if(__any_sync(0xffffffffu, want && !got)) more = false;      // global counter ran past the end
				else pool_ahead(pool, a.task_ctr64, a.chunk);
			} else if(want) mode = M_DONE;
		}
		if(!__any_sync(0xffffffffu, mode != M_DONE)) break;
		// ---------------- single fetch point ----------------
		// Every lane picks the address of the one 16-byte (aligned) piece it needs -- whatever table its walk is at -- plus
		// a second rank16 entry when a range straddles two 64-row blocks; then ONE predicated load instruction serves all
		// lanes (and one more the straddlers), and 2 + 2 RW more the lanes whose read arrives.  Left to the compiler, each
		// table's load sank into the branch that consumes it, and a warp then paid one memory latency per table in play
		// instead of one per trip (ncu: stalls at the K-mer-table consumer with 4 of 32 lanes active).
		int c = 4;
		const bool lf = mode == M_LF, task = mode == M_TASK;
		bool range = false, jump = false, known_fail = false;
		const void* p0 = nullptr; const void* p1 = nullptr; uint32_t sub = 0;
		if(mode == M_FTAB) { p0 = ftab2 + fi; if(REQS) q_f2++; }                                // (top, bot) of the 10-mer
		else if(mode == M_FTABK) { p0 = ftabk + (fi & ((1ull << (2 * fk)) - 1ull)); if(REQS) q_fk++; }   // range + death bitmap of the K-mer
		else if(lf) {
			c = rd.base(dep);
			if(c <= 3) {
				range = (bot - top) != 1;
				const uint64_t width = bot - top;
				if(dep == fail_at && !range) known_fail = true;      // the walk8 entry already said that this step of the single row fails: no request
				else if(w8 && dep >= slow_until && rlen - dep >= 8 && bot <= a.v.walk8_rows) {
					// Eight steps in one gather: the read's next eight bases are the ones stored for the range's first AND last
					// row.  Then the range after them is exactly [W8(top), W8(bot - 1) + 1), whatever the rows in between do
					// (cf_logic.h, walk8_steps).  One 16-byte piece serves both ends when they share it.
					jump = true; p0 = w8 + (top & ~1ull); sub = (uint32_t)(top & 1);
					if(range) { const uint64_t last = bot - 1; sub |= (uint32_t)(last & 1) << 1; if((last & ~1ull) != (top & ~1ull)) p1 = w8 + (last & ~1ull); }
					if(REQS) { q_w8 += p1 ? 2 : 1; if(range) j_rng++; else j_row++; }
				} else {
					p0 = r16 + r16_entry(top, c);                           // (occ, bits): one request per rank query
					if(range && (bot >> 6) != (top >> 6)) p1 = r16 + r16_entry(bot, c);
					if(REQS) { const uint32_t n = p1 ? 2 : 1; q_r16 += n; if(width == 1) q_w1 += n; else if(width <= 4) q_w24 += n; else q_w5 += n; }
				}
			}
		}
		const uint32_t unit = tid >> msh, mate = (tid >> 1) & (msh - 1u);
		const uint64_t* tpk = a.pk + (size_t)tid * a.W; const uint32_t* tnm = a.nm + (size_t)tid * a.W;
		uint32_t fl = 3;
		if(REQS) { if(p0) s_lreq++; t_issue = clock64(); }
		// the second piece lands in registers of its own: copied from the first before its load (so that lanes without a second
		// piece find the first there), the copy waited for the first load and the warp's second pieces went out one round trip late
		const bool two = p1 != nullptr;
		ulonglong2 e = make_ulonglong2(0, 0), e2 = make_ulonglong2(0, 0);
		ld_if(e, p0);
		ld_if(e2, p1);
		ld_if(rlen, (mate ? a.b.len[1] : a.b.len[0]) + unit, task);      // no runtime index into the parameter arrays
		ld_if(fl, a.b.flags + unit, task && a.b.flags != nullptr);
		#pragma unroll
		for(int k = 0; k < RW; k++) { ld_if(rd.rw[k], tpk + k, task && (uint32_t)k < a.W); ld_if(rd.nw[k], tnm + k, task && (uint32_t)k < a.W); }
		if(REQS) {      // a vote on the loaded values: the clock after it is read when every load of the warp has landed
			if(__any_sync(0xffffffffu, (e.x ^ e2.y ^ rd.rw[RW - 1] ^ rd.nw[RW - 1] ^ rlen ^ fl) == 0x9e3779b97f4a7c15ull)) s_task += 1ull << 40;
			t_data = clock64();
		}
		// ---------------- consume ----------------
		// ended: the partial search is over and its hit is (h_top, h_bot, hl) at `offset`, with cur already behind it;
		// stop: it is over where the walk stands (top, bot, dep); fresh: the lane's read has just arrived
		const ulonglong2 tq = e, bq = two ? e2 : e;
		bool ended = false, stop = false, fresh = false;
		uint64_t h_top = kOff, h_bot = kOff; uint32_t hl = 0;
		if(task) {
			if(REQS) paths |= 1u;
			#pragma unroll
			for(int k = 0; k < RW; k++) if((uint32_t)k >= a.W) { rd.rw[k] = 0; rd.nw[k] = 0; }
			nh = 0; nt = 0;
			if(!((fl >> mate) & 1) || rlen == 0) { a.nhits[tid] = 0; mode = M_NEED; }          // filtered mate: asks again in the next trip
			else { cur = 0; slow_until = 0; fail_at = 0xffffffffu; nolong = true; fresh = true; }
		} else if(mode == M_FTABK) {
			if(REQS) paths |= 2u;
			const uint32_t ext = (uint32_t)(fi >> (2 * fk));
			const uint32_t dv = ext ? ftabk_death(e.y, ext & 63u) : 0u;
			const uint64_t width = e.x >> 40;
			if(dv) {                                      // the range dies after K + dv - 1 bases: that is the hit partialSearch reports
				hl = fk + dv - 1u; h_top = h_bot = kUnk; cur += hl; ended = true;
			} else if(width != 0 && width != kFtabkWide) {   // same state partialSearch reaches after K bases
				top = e.x & kRowMask; bot = top + width; dep = cur + fk;
				if(dep < rlen) mode = M_LF; else stop = true;
			} else { fi &= (1ull << (2 * fc)) - 1ull; mode = M_FTAB; }   // died between base fc and K, or too wide: replay from the 10-mer
		} else if(mode == M_FTAB) {
			if(REQS) paths |= 4u;
			top = e.x; bot = e.y;
			dep = cur + fc;
			if(bot <= top) { hl = dep - offset; cur = dep; ended = true; }      // hi_aligner.h:971-982
			else if(dep < rlen) mode = M_LF;
			else stop = true;
		} else if(jump) {
			if(REQS) paths |= 8u;
			uint64_t win; uint32_t nwin; rd.window(dep, win, nwin);
			const uint64_t w = (sub & 1u) ? e.y : e.x;                       // entry of the first row
			const uint64_t wl = range ? ((sub & 2u) ? bq.y : bq.x) : w;      // entry of the last row
			const uint32_t st = walk8_steps(w, win, nwin), sb = range ? walk8_steps(wl, win, nwin) : st;
			if((st & sb) == 8u) {                                            // both end rows follow all eight bases
				if(REQS) { if(range) j_rng_ok++; else j_row_ok++; if(bot - top >= 5) j_w5_ok++; }
				top = w & kWalkRowMask; bot = (wl & kWalkRowMask) + 1; dep += 8;
				stop = dep >= rlen;
			} else {      // an end row leaves within the next eight steps: take them one by one until both failing ends have left
				slow_until = dep + walk8_retry(st, sb);
				if(!range) fail_at = dep + st;      // a single row: the entry tells which step ends the hit (no request for it)
			}
		} else if(lf) {
			if(REQS) paths |= 16u;
			bool fail = c > 3 || known_fail;
			uint64_t t = 0, b = 0;
			if(!fail) {
				t = r16_lf(a.v, top, c, tq.x, tq.y);
				if(range) b = r16_lf(a.v, bot, c, bq.x, bq.y);
				else {                                    // mapLF1 bt2_idx.h:2910-2933: BWT[top] must be c ('$' has no bit)
					if(!((tq.y >> (top & 63)) & 1ull)) fail = true;
					b = t + 1;
				}
				if(b <= t) fail = true;
			}
			if(fail) stop = true;
			else { top = t; bot = b; dep++; stop = dep >= rlen; }
		}
		if(stop) { h_top = top; h_bot = bot; hl = dep - offset; cur = dep; ended = true; }
		// ---------------- restart ----------------
		// The hit store, then searchForwardAndReverse's restart policy (classifier.h:686-766), then partialSearch's prologue
		// (hi_aligner.h:939-982) at `cur`, which ends in M_FTABK / M_FTAB (fi set) or, on an N inside the first 10-mer or with
		// fewer than 10 bases left, in another hit -- hence a loop.  A lane leaves it searching or in M_NEED with its nhits word stored.
		#pragma unroll 1
		while(ended || fresh) {
			if(ended) {
				if(REQS) paths |= 1u << 16;
				if(a.keep_short || hl >= kLongLen) {
					if(nh < a.cap) { HitRec* h = a.hits + (size_t)tid * a.cap + nh; h->top = h_top; h->bot = h_bot; h->bwoff = offset; h->len = hl; }
					else atomicExch(a.overflow, 1u);
					nh++;
				}
				nt++;
				if(hl >= a.p.min_hitlen) nolong = false;
				ended = false;
				bool done = cur >= rlen;
				if(!done) { if(hl > a.p.increment) cur += 1; if(cur + a.p.min_hitlen >= rlen) done = true; }
				if(done) { a.nhits[tid] = nh_pack(nh, nt, nolong); mode = M_NEED; break; }
			}
			if(REQS) paths |= 1u << 18;
			fresh = false;
			offset = cur; h_top = h_bot = kOff;
			if(rlen - cur < fc) { hl = rlen - cur; cur = rlen; ended = true; continue; }      // too short for the 10-mer table: the rest is one hit
			uint64_t win; uint32_t nwin; rd.window(cur, win, nwin);
			const uint32_t nbits = nwin & ((1u << fc) - 1u);
			if(nbits) { hl = (uint32_t)__ffs(nbits); cur += hl; ended = true; continue; }
			if(fk && rlen - cur >= fk && !(nwin & ((1u << fk) - 1u))) {
				fi = win & ((1ull << (2 * fk)) - 1ull);
				if(fd && rlen - cur >= fd && !(nwin & ((1u << fd) - 1u))) fi |= (64ull | ((win >> (2 * fk)) & 63ull)) << (2 * fk);
				mode = M_FTABK;
			} else {
				fi = win & ((1ull << (2 * fc)) - 1ull);
				mode = M_FTAB;
			}
		}
		if(REQS) {
			const uint32_t all = __reduce_or_sync(0xffffffffu, paths);
			s_trips++; s_cons += __popc(all & 0xffffu); s_rest += __popc(all >> 16); if(all & (1u << 17)) s_task++;
			const long long t_end = clock64(); s_head += t_issue - t_top; s_wait += t_data - t_issue; s_tail += t_end - t_data;
		}
	}
	if(REQS && a.ctr) {
		atomicAdd(&a.ctr->req_rank16, q_r16); atomicAdd(&a.ctr->req_ftab2, q_f2); atomicAdd(&a.ctr->req_ftabk, q_fk); atomicAdd(&a.ctr->req_walk8, q_w8);
		atomicAdd(&a.ctr->r16_w1, q_w1); atomicAdd(&a.ctr->r16_w2_4, q_w24); atomicAdd(&a.ctr->r16_w5, q_w5);
		atomicAdd(&a.ctr->w8_try_row, j_row); atomicAdd(&a.ctr->w8_ok_row, j_row_ok); atomicAdd(&a.ctr->w8_try_range, j_rng); atomicAdd(&a.ctr->w8_ok_range, j_rng_ok); atomicAdd(&a.ctr->w8_ok_w5, j_w5_ok);
		atomicAdd(&a.ctr->it_lane_req, s_lreq);
		if((threadIdx.x & 31) == 0) {
			atomicAdd(&a.ctr->it_warp, s_trips); atomicAdd(&a.ctr->it_consumers, s_cons); atomicAdd(&a.ctr->it_restarts, s_rest); atomicAdd(&a.ctr->it_task, s_task & ((1ull << 40) - 1ull));
			atomicAdd(&a.ctr->clk_head, s_head); atomicAdd(&a.ctr->clk_wait, s_wait); atomicAdd(&a.ctr->clk_tail, s_tail);
		}
	}
}

// =======================================================================================
// k_prep / k_rows / k_score (thread per unit)
// =======================================================================================
struct UnitArgs {
	IndexView v; Params p; BatchView b;
	HitRec* hits; uint32_t* nhits; uint32_t cap;
	uint32_t* nrows;            // per unit
	uint64_t* row_off;          // per unit: where its rows (ids, hit-map scratch, sparse records) start; handed out by k_prep
	unsigned long long* row_total;   // allocation counter = total rows of the batch
	uint64_t* rows; uint32_t* ids; uint64_t rows_cap;
	Entry* entries; TaxCnt* tcs; OutRec* recs_sparse; uint32_t* nout;
	unsigned int* overflow;
	Counters* ctr;
	HitRec* regen; uint32_t* regen_n; unsigned long long* regen_ctr; uint64_t regen_slots; uint32_t full_cap; uint32_t keep_short;
};

// One strand's whole greedy search by a single thread, with the device tables: the hits search_strand_scalar (cf_logic.h, the
// twin the CPU tests pin against the oracle) would produce, but reached the way k_search_t reaches them -- K-mer jump, one
// rank16 entry per step when top and bot share a block, eight bases per walk8 gather of the range's end rows -- so that regenerating
// a list costs ~30 dependent gathers instead of ~250.  Used by k_prep (lists whose short hits matter) and k_search_long.
// One partial search from `cur` (partial_search_scalar's result) with the device tables.  CR: on the compact rank layout (v.cr)
// every LF step is cr_lf, and *nreq (when given) counts its 32-byte sector pieces.  Callers pick the instantiation once per
// kernel or walk, so the rank16 one is the walk it always was.
template <bool CR>
__device__ __forceinline__ void partial_search_dev(const IndexView& v, const uint8_t* fw, uint32_t len, int strand, uint32_t cur,
                                                   HitRec& h, uint32_t& new_cur, bool& done, unsigned long long* nreq = nullptr) {
	const ulonglong2* r16 = reinterpret_cast<const ulonglong2*>(v.rank16);
	const ulonglong2* ftab2 = reinterpret_cast<const ulonglong2*>(v.ftab2);
	const ulonglong2* ftabk = reinterpret_cast<const ulonglong2*>(v.ftabk);
	const uint32_t fc = (uint32_t)v.ftab_chars, fk = v.ftabk ? (uint32_t)v.ftabk_chars : 0u;
	auto base = [&](uint32_t d) -> int { return seq_at(fw, len, strand, len - 1 - d); };     // the base consumed at search depth d
	{
		h.bwoff = cur; done = false;
		const uint32_t offset = cur;
		if(len - cur < fc) { h.top = h.bot = kOff; h.len = len - offset; new_cur = len; done = true; }
		else {
			uint32_t firstn = 0xffffffffu; uint64_t fi = 0;
			const uint32_t span = (fk && len - cur >= fk) ? fk : fc;
			for(uint32_t i = 0; i < span; i++) { const int c = base(cur + i); if(c > 3) { firstn = i; break; } fi |= (uint64_t)c << (2 * i); }
			if(firstn < fc) { new_cur = cur + firstn + 1; h.top = h.bot = kOff; h.len = new_cur - offset; done = new_cur >= len; }
			else {
				uint64_t top = 0, bot = 0; uint32_t dep = 0; bool have = false;
				if(span == fk && fk > fc && firstn == 0xffffffffu) {      // the range only: regenerated lists need exact ranges
					const uint64_t x = __ldg(&ftabk[fi].x), width = x >> 40;
					if(width != 0 && width != kFtabkWide) { top = x & kRowMask; bot = top + width; dep = cur + fk; have = true; }
				}
				if(!have) { const ulonglong2 e = __ldg(ftab2 + (fi & ((1ull << (2 * fc)) - 1ull))); top = e.x; bot = e.y; dep = cur + fc; }
				if(bot <= top) { h.top = h.bot = kOff; h.len = dep - offset; new_cur = dep; done = dep >= len; }
				else {
					uint32_t slow_until = 0;
					while(dep < len) {
						const int c = base(dep);
						if(c > 3) break;
						if(v.walk8 && bot <= v.walk8_rows && len - dep >= 8 && dep >= slow_until) {     // eight bases in one gather (k_search_t's rule)
							uint64_t win = 0; uint32_t nwin = 0;
							for(uint32_t j = 0; j < 8; j++) { const int b = base(dep + j); if(b > 3) nwin |= 1u << j; else win |= (uint64_t)b << (2 * j); }
							const uint64_t et = __ldg(v.walk8 + top), eb = bot - top == 1 ? et : __ldg(v.walk8 + bot - 1);
							const uint32_t st = walk8_steps(et, win, nwin), sb = walk8_steps(eb, win, nwin);
							if((st & sb) == 8u) { top = et & kWalkRowMask; bot = (eb & kWalkRowMask) + 1; dep += 8; continue; }
							slow_until = dep + walk8_retry(st, sb);
						}
						if(CR) {
							if(nreq) *nreq += 1 + ((top % kCrRows) > 64) + (bot - top == 1 ? 0 : 1 + ((bot % kCrRows) > 64));
							if(bot - top == 1) {
								if(top == v.zoff || cr_bwt(v, top) != c) break;            // mapLF1: BWT[top] must be c, and not the '$' stored as A
								top = cr_lf(v, top, c); bot = top + 1; dep++;
							} else {
								const uint64_t t = cr_lf(v, top, c), b = cr_lf(v, bot, c);
								if(b <= t) break;
								top = t; bot = b; dep++;
							}
							continue;
						}
						if(bot - top == 1) {
							const ulonglong2 e = __ldg(r16 + r16_entry(top, c));
							if(!((e.y >> (top & 63)) & 1ull)) break;                      // mapLF1: BWT[top] must be c ('$' has no bit)
							top = r16_lf(v, top, c, e.x, e.y); bot = top + 1; dep++;
						} else {
							const ulonglong2 et = __ldg(r16 + r16_entry(top, c));
							const ulonglong2 eb = (bot >> 6) == (top >> 6) ? et : __ldg(r16 + r16_entry(bot, c));
							const uint64_t t = r16_lf(v, top, c, et.x, et.y), b = r16_lf(v, bot, c, eb.x, eb.y);
							if(b <= t) break;
							top = t; bot = b; dep++;
						}
					}
					h.top = top; h.bot = bot; h.len = dep - offset; new_cur = dep; done = dep >= len;
				}
			}
		}
	}
}
template <bool CR>
__device__ uint32_t search_strand_dev(const IndexView& v, const Params& p, const uint8_t* fw, uint32_t len, int strand, HitRec* hits, uint32_t cap,
                                      unsigned long long* nreq = nullptr) {
	uint32_t cur = 0, n = 0;
	if(len == 0) return 0;
	for(;;) {
		HitRec h; uint32_t new_cur; bool done;
		partial_search_dev<CR>(v, fw, len, strand, cur, h, new_cur, done, nreq);
		if(n < cap) hits[n] = h;
		n++;
		cur = new_cur;
		if(done) break;
		if(h.len > p.increment) cur += 1;
		if(cur + p.min_hitlen >= len) break;
	}
	return n;
}

// k_search_long: batches with a read longer than k_search_t's widest register window (kWindowLen bases).  One thread per
// (unit, mate, strand) task runs the strand's whole search from the byte form of the read and stores every hit, so k_prep
// never regenerates these lists.  SCALAR runs search_strand_scalar, one LF step at a time with the jump tables off, for every read
// length: the pass that counts the reference's operations (SURVEY 8d).  On rank16 the table walk counts no load requests for these
// reads; on the compact rank layout, where this kernel serves every read length, CFB_COUNT=2 counts its sector pieces in req_rank16.
static const uint32_t kWindowLen = 320;      // 10 register words of 32 bases
template <bool SCALAR, bool CR = false>
__global__ void __launch_bounds__(kSearchThreads) k_search_long(const SearchArgs a) {
	const uint32_t per = 2u * (uint32_t)a.b.n_mates;
	Counters local; memset(&local, 0, sizeof local);
	unsigned long long* nreq = !SCALAR && CR && a.ctr ? &local.req_rank16 : nullptr;
	for(uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x; tid < a.ntasks; tid += gridDim.x * blockDim.x) {
		const uint32_t unit = tid / per, rem = tid - unit * per;
		const int mate = (int)(rem >> 1), strand = (int)(rem & 1);
		const uint8_t fl = a.b.flags ? a.b.flags[unit] : 3;
		const uint32_t len = a.b.len[mate][unit];
		if(!((fl >> mate) & 1) || len == 0) { a.nhits[tid] = 0; continue; }
		const uint8_t* fw = a.b.bases + a.b.off[mate][unit];
		HitRec* hits = a.hits + (size_t)tid * a.cap;
		const uint32_t n = SCALAR ? search_strand_scalar(a.v, a.p, fw, len, strand, hits, a.cap, &local)
		                          : search_strand_dev<CR>(a.v, a.p, fw, len, strand, hits, a.cap, nreq);
		if(n > a.cap) atomicExch(a.overflow, 1u);      // the host grows the lists and re-runs the batch
		a.nhits[tid] = nh_pack(min(n, a.cap), n, false);
	}
	if(SCALAR && a.ctr) {
		atomicAdd(&a.ctr->partial_searches, local.partial_searches); atomicAdd(&a.ctr->ftab_probes, local.ftab_probes);
		atomicAdd(&a.ctr->sides_search, local.sides_search); atomicAdd(&a.ctr->lf_steps, local.lf_steps);
	}
	if(nreq && local.req_rank16) atomicAdd(&a.ctr->req_rank16, local.req_rank16);
}

typedef void (*SearchKernel)(const SearchArgs);
// count 1: the scalar search, which counts the reference's operations; otherwise the thread-per-walk kernel whose register
// window holds the batch's longest read (count 2: its request-counting instantiation).  k_search_t reads rank16 only: on the
// compact rank layout every batch takes the thread-per-walk kernel.
static SearchKernel search_kernel(uint32_t maxlen, int count, bool compact) {
	if(count == 1) return k_search_long<true>;
	if(compact) return k_search_long<false, true>;
	if(maxlen > kWindowLen) return k_search_long<false>;
	const bool reqs = count == 2;
	if(maxlen > 160) return reqs ? k_search_t<true, 10> : k_search_t<false, 10>;
	if(maxlen > 128) return reqs ? k_search_t<true, 5> : k_search_t<false, 5>;      // 2 x 150 bp runs
	return reqs ? k_search_t<true, 4> : k_search_t<false, 4>;
}

// found[r][st] receives the number of hits the search found for the list (0 for a regenerated list); tpos[r] the index of
// the mate's first nhits word
__device__ __forceinline__ bool load_unit(const UnitArgs& a, uint32_t unit, UnitHits& u, const uint8_t* fw[2], uint32_t found[2][2], size_t tpos[2]) {
	const uint8_t fl = a.b.flags ? a.b.flags[unit] : 3;
	u.n_mates = 0;
	for(int m = 0; m < a.b.n_mates; m++) {
		if(!((fl >> m) & 1)) continue;
		const uint32_t len = a.b.len[m][unit];
		if(len == 0) continue;
		const int r = u.n_mates++;
		const size_t t0 = ((size_t)unit * a.b.n_mates + m) * 2;
		u.rdlen[r] = len; fw[r] = a.b.bases + a.b.off[m][unit]; tpos[r] = t0;
		const uint32_t raw[2] = {a.nhits[t0], a.nhits[t0 + 1]};
		for(int st = 0; st < 2; st++) {
			if(raw[st] & kListRegen) {                            // regenerated by an earlier k_prep pass over this batch
				const uint32_t slot = raw[st] & 0x3fffffffu;
				u.L[r][st] = a.regen + (size_t)slot * a.full_cap; u.n[r][st] = a.regen_n[slot]; found[r][st] = 0;
			} else {
				u.L[r][st] = a.hits + (t0 + st) * a.cap; u.n[r][st] = min(nh_stored(raw[st]), a.cap); found[r][st] = nh_found(raw[st]);
			}
		}
		for(int st = 0; st < 2; st++) if(list_dropped(raw, st)) u.n[r][st] = 0;
	}
	return u.n_mates > 0;
}

// thread per unit: post-process + sort the hit lists, count the SA rows to resolve, take a slice of the row buffer
// (one atomic per warp) and write the rows with the scoring plan in their high bits.  EMIT_ONLY re-does only the last
// two steps on lists that are already final (after the row buffer had to grow).
template <int MINB, bool EMIT_ONLY>
__global__ void __launch_bounds__(128, MINB) k_prep(const UnitArgs a) {
	const uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x;
	const bool live = unit < a.b.n_units;
	UnitHits u; const uint8_t* fw[2]; uint32_t found[2][2]; size_t tpos[2];
	uint64_t rows = 0; bool have = false;
	if(live && (have = load_unit(a, unit, u, fw, found, tpos))) {
		if(EMIT_ONLY) { CountRows cr(a.p, u); for_each_visit(a.p, u, cr); rows = cr.rows; }
		else {
			Counters local; Counters* lc = nullptr;
			if(a.ctr) { memset(&local, 0, sizeof local); lc = &local; }
			// Only the long hits were stored (see kListRegen): where the short ones can matter, run the strand's search again
			// on this thread (search_strand_dev) into the side buffer, and let the list point there from now on.
			if(!a.keep_short) for(int r = 0; r < u.n_mates; r++) {
				for(int st = 0; st < 2; st++) {
					if(!list_needs_regen(u.n[r][st], u.n[r][st ^ 1], found[r][st])) continue;
					const unsigned long long slot = atomicAdd(a.regen_ctr, 1ull);
					if(slot >= a.regen_slots) { atomicExch(a.overflow, 4u); continue; }      // the host grows the side buffer and re-runs the batch
					HitRec* L = a.regen + (size_t)slot * a.full_cap;
					const uint32_t n = a.v.cr ? search_strand_dev<true>(a.v, a.p, fw[r], u.rdlen[r], st, L, a.full_cap)
					                          : search_strand_dev<false>(a.v, a.p, fw[r], u.rdlen[r], st, L, a.full_cap);
					if(n > a.full_cap) atomicExch(a.overflow, 1u);
					u.L[r][st] = L; u.n[r][st] = min(n, a.full_cap);
					a.regen_n[slot] = u.n[r][st]; a.nhits[tpos[r] + st] = kListRegen | (uint32_t)slot;
				}
			}
			// Hits the death bitmap ended carry no SA range.  Where a short hit's range can matter -- twin removal, introsort's
			// tie permutation, or the time stamps of counted hits shorter than kLongLen (list_needs_exact_ranges) -- recompute
			// the ranges, exactly as partialSearch would.
			for(int r = 0; r < u.n_mates; r++) {
				for(int st = 0; st < 2; st++) {
					if(!list_needs_exact_ranges(a.p, u.L[r][st], u.n[r][st], u.n[r][st ^ 1])) continue;
					for(uint32_t i = 0; i < u.n[r][st]; i++) {
						HitRec& h = u.L[r][st][i];
						if(h.top != kUnk) continue;
						HitRec t; uint32_t nc; bool dn;
						partial_search_scalar(a.v, fw[r], u.rdlen[r], st, h.bwoff, t, nc, dn, nullptr);
						h.top = t.top; h.bot = t.bot;
					}
				}
			}
			for(int r = 0; r < u.n_mates; r++) post_search(a.v, a.p, fw[r], u.rdlen[r], u.L[r][0], u.n[r][0], u.L[r][1], u.n[r][1], lc);
			SortAndCount sc(a.p, u);
			for_each_visit(a.p, u, sc);
			rows = sc.rows;
			if(lc) {
				atomicAdd(&a.ctr->units, 1ull);
				if(local.ext_searches) {
					atomicAdd(&a.ctr->ext_searches, local.ext_searches); atomicAdd(&a.ctr->partial_searches, local.partial_searches);
					atomicAdd(&a.ctr->ftab_probes, local.ftab_probes); atomicAdd(&a.ctr->sides_search, local.sides_search); atomicAdd(&a.ctr->lf_steps, local.lf_steps);
				}
			}
		}
		if(rows > 0xFFFFFFFFull) rows = 0xFFFFFFFFull;
	}
	const unsigned lane = threadIdx.x & 31;
	uint64_t incl = rows;
	for(int d = 1; d < 32; d <<= 1) { const uint64_t t = __shfl_up_sync(0xffffffffu, incl, d); if((int)lane >= d) incl += t; }
	const uint64_t warp_total = __shfl_sync(0xffffffffu, incl, 31);
	unsigned long long base = 0;
	if(lane == 31 && warp_total) base = atomicAdd(a.row_total, (unsigned long long)warp_total);
	base = __shfl_sync(0xffffffffu, base, 31);
	if(!live) return;
	const uint64_t off = base + incl - rows;
	a.nrows[unit] = (uint32_t)rows; a.row_off[unit] = off;
	if(rows && off + rows <= a.rows_cap) { EmitRows er(a.p, u, a.rows + off); for_each_visit(a.p, u, er); }   // else: the host grows the buffer and re-runs EMIT_ONLY
}

// k_prep hands out row slices per warp, so the rows of a warp's 32 units form one contiguous span.  A warp whose span fits
// what is left of its CTA's pool keeps its units' hit maps there, each at the unit's own offset inside the span (nmap <= n
// bounds them); a warp whose span does not fit keeps them in the global scratch at the units' row offsets.  Only the hit maps
// live in the pool: rows and ids are read where k_prep and k_lookup left them, records go straight to the sparse buffer, and the
// tree reduction's TaxCnt scratch (a fraction of a percent of the units run it) is always the global one.  A span averages
// ~80 rows on the bench batch (2.4 rows per unit), so what decides how many warps the pool takes is the bytes per row.
static const int kScoreThreads = 128;
static const uint32_t kScorePool = 232;       // hit-map entries per CTA: 14.5 KB, as much shared memory as the earlier pool of 128 rows of 116 bytes, which 256 rows (29 KB) beat in k_score but lost to in e2e, where k_score shares SMs with search kernels (measured)
static const uint32_t kNoSlot = 0xffffffffu;
__device__ __forceinline__ uint32_t log2_bucket(uint64_t x) { const uint32_t b = 63u - (uint32_t)__clzll((long long)x); return b < 7u ? b : 7u; }     // x >= 1
// COUNT: the instantiation of the counting passes, which also fills the sc_* counters (how the rows, distinct ids and tree
// reductions of the batch are distributed, and how many warps the shared pool could not take)
template <int MINB, bool COUNT>
__global__ void __launch_bounds__(kScoreThreads, MINB) k_score(const UnitArgs a) {
	__shared__ Entry s_map[kScorePool];
	__shared__ uint32_t s_used;
	if(threadIdx.x == 0) s_used = 0;
	__syncthreads();
	const uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x;
	const unsigned lane = threadIdx.x & 31;
	const bool valid = unit < a.b.n_units;
	const bool fits = *a.row_total <= a.rows_cap;          // else the host grows the row buffer and runs the batch's tail again
	const uint64_t n = valid && fits ? a.nrows[unit] : 0, off = valid && fits ? a.row_off[unit] : 0;
	const uint64_t base = __shfl_sync(0xffffffffu, off, 0);        // lane 0's unit is the warp's first: its slice starts the span
	uint64_t span = n ? off + n - base : 0;
	for(int d = 16; d > 0; d >>= 1) span = max(span, __shfl_xor_sync(0xffffffffu, span, d));
	uint32_t slot = kNoSlot;
	if(lane == 0 && span) {
		uint32_t cur = *(volatile uint32_t*)&s_used;
		while(span <= kScorePool - cur) {
			const uint32_t old = atomicCAS(&s_used, cur, cur + (uint32_t)span);
			if(old == cur) { slot = cur; break; }
			cur = old;
		}
	}
	slot = __shfl_sync(0xffffffffu, slot, 0);
	const bool sh = slot != kNoSlot;
	uint32_t no = 0;
	if(n > 0) {
		const uint8_t fl = a.b.flags ? a.b.flags[unit] : 3;
		int mates = 0;
		for(int m = 0; m < a.b.n_mates; m++) if(((fl >> m) & 1) && (m ? a.b.len[1][unit] : a.b.len[0][unit]) != 0) mates++;
		Entry* map = sh ? s_map + slot + (uint32_t)(off - base) : a.entries + off;
		const uint32_t nmap = score_plan(a.v, a.p, a.rows + off, a.ids + off, n, map);
		uint32_t rounds = 0;
		no = reduce_and_emit(a.v, a.p, mates == 2, map, nmap, a.tcs + off, a.recs_sparse + off, COUNT ? &rounds : nullptr);
		if(COUNT) {
			atomicAdd(&a.ctr->sc_units, 1ull); atomicAdd(&a.ctr->sc_rows, (unsigned long long)n); atomicAdd(&a.ctr->sc_nmap, (unsigned long long)nmap);
			atomicAdd(&a.ctr->sc_rows_hist[log2_bucket(n)], 1ull);
			if(nmap) atomicAdd(&a.ctr->sc_nmap_hist[log2_bucket(nmap)], 1ull);
			if(rounds) { atomicAdd(&a.ctr->sc_reduce, 1ull); atomicAdd(&a.ctr->sc_rounds, (unsigned long long)rounds); }
		}
	}
	if(COUNT && lane == 0 && span) { atomicAdd(&a.ctr->sc_warps, 1ull); if(!sh) atomicAdd(&a.ctr->sc_warps_global, 1ull); }
	if(valid) a.nout[unit] = no;
}

// =======================================================================================
// scan (u32 -> exclusive u64, n+1 outputs) : 3 small kernels, 1024 elements per block
// =======================================================================================
static const int kScanBlock = 256, kScanPer = 4;   // 1024 per block

__global__ void __launch_bounds__(kScanBlock) k_scan_sums(const uint32_t* in, uint64_t n, uint64_t* bsum) {
	__shared__ uint64_t sh[kScanBlock];
	const uint64_t base = (uint64_t)blockIdx.x * kScanBlock * kScanPer + (uint64_t)threadIdx.x * kScanPer;
	uint64_t s = 0;
	for(int i = 0; i < kScanPer; i++) if(base + i < n) s += in[base + i];
	sh[threadIdx.x] = s; __syncthreads();
	for(int d = kScanBlock / 2; d > 0; d >>= 1) { if((int)threadIdx.x < d) sh[threadIdx.x] += sh[threadIdx.x + d]; __syncthreads(); }
	if(threadIdx.x == 0) bsum[blockIdx.x] = sh[0];
}
__global__ void k_scan_top(uint64_t* bsum, uint64_t nb, uint64_t* total) {   // single thread block, serial over blocks by chunks
	__shared__ uint64_t carry;
	__shared__ uint64_t sh[1024];
	if(threadIdx.x == 0) carry = 0;
	__syncthreads();
	for(uint64_t base = 0; base < nb; base += 1024) {
		const uint64_t i = base + threadIdx.x;
		const uint64_t vv = i < nb ? bsum[i] : 0;
		sh[threadIdx.x] = vv; __syncthreads();
		for(int d = 1; d < 1024; d <<= 1) { uint64_t t = (int)threadIdx.x >= d ? sh[threadIdx.x - d] : 0; __syncthreads(); sh[threadIdx.x] += t; __syncthreads(); }
		if(i < nb) bsum[i] = carry + sh[threadIdx.x] - vv;
		__syncthreads();
		if(threadIdx.x == 1023) carry += sh[1023];
		__syncthreads();
	}
	if(threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(kScanBlock) k_scan_apply(const uint32_t* in, uint64_t n, const uint64_t* bsum, const uint64_t* total, uint64_t* out) {
	__shared__ uint64_t sh[kScanBlock];
	const uint64_t base = (uint64_t)blockIdx.x * kScanBlock * kScanPer + (uint64_t)threadIdx.x * kScanPer;
	uint32_t vals[kScanPer]; uint64_t s = 0;
	for(int i = 0; i < kScanPer; i++) { vals[i] = base + i < n ? in[base + i] : 0; s += vals[i]; }
	sh[threadIdx.x] = s; __syncthreads();
	for(int d = 1; d < kScanBlock; d <<= 1) { uint64_t t = (int)threadIdx.x >= d ? sh[threadIdx.x - d] : 0; __syncthreads(); sh[threadIdx.x] += t; __syncthreads(); }
	uint64_t run = bsum[blockIdx.x] + sh[threadIdx.x] - s;
	for(int i = 0; i < kScanPer; i++) { if(base + i < n) out[base + i] = run; run += vals[i]; }
	if(blockIdx.x == 0 && threadIdx.x == 0) out[n] = *total;
}

// =======================================================================================
// SA row -> sequence id
// =======================================================================================
enum { R_DONE = 0, R_WALK = 1, R_SAMPLE = 2, R_NEED = 3 };
struct ResolveArgs {
	IndexView v; const uint64_t* rows; uint32_t* ids; uint16_t* ids16; const uint64_t* total; uint64_t rows_cap;
	unsigned long long* task_ctr; uint32_t chunk; Counters* ctr;
};
// One LF step of a 4-lane group (k_resolve_c, k_build_walk8): lane j holds base j's rank16 entry `e` of row's block; the lane
// whose indicator bit is set at the row owns BWT[row] and its LF value is the next row.  Returns that base, or -1 where no lane
// owns the row (the '$' row; `next` is then meaningless).
__device__ __forceinline__ int group_lf(const IndexView& v, uint64_t row, const ulonglong2 e, uint64_t& next) {
	const unsigned gl = threadIdx.x & 3, gbase = threadIdx.x & 28, gmask = 0xFu << gbase;
	const uint64_t mine = r16_lf(v, row, (int)gl, e.x, e.y);
	const int src = __ffs((__ballot_sync(gmask, (e.y >> (row & 63)) & 1ull) >> gbase) & 0xFu) - 1;
	next = __shfl_sync(gmask, mine, gbase + (src < 0 ? 0 : src));
	return src;
}

// ---------------------------------------------------------------------------------------
// k_resolve_c: 4 lanes per SA row over rank16.  Lane j fetches the entry of base j, so the 64-byte
// chunk of a block arrives with ONE load request per walk step; the lane whose indicator bit is set
// at the row knows BWT[row] and its own LF value is the next row.  The genome-boundary prefilter is the
// flag bit in A's occ word (no separate bitmap load).
// ---------------------------------------------------------------------------------------
// IDENT: rows are 0..n-1 themselves and results go to the (16- or 32-bit) resolve table -- used once at index load.
// CR: the compact rank layout.  The four lanes of a group step together through cr_bwt / cr_lf of the same row (their loads
// coalesce), and boundary rows are found through the .4.cf bitmap (bbits), as rank16's boundary flag has no place there.
template <bool COUNT, bool IDENT, bool CR = false>
__global__ void __launch_bounds__(kSearchThreads) k_resolve_c(const ResolveArgs a) {
	const unsigned lane = threadIdx.x & 31, gl = lane & 3, gbase = lane & 28, gmask = 0xFu << gbase;
	const ulonglong2* r16 = reinterpret_cast<const ulonglong2*>(a.v.rank16);
	uint64_t n = *a.total; if(n > a.rows_cap) return;          // the row buffer was too small: slices have holes, the host re-runs the batch
	const uint64_t lowmask = ((uint64_t)1 << a.v.off_rate) - 1;
	uint64_t idx = 0, row = 0;
	int mode = R_NEED;
	unsigned long long c_walk = 0, c_rows = 0;
	WarpPool pool;
	bool more = true;
	auto put = [&](uint32_t v) { if(IDENT && a.ids16) a.ids16[idx] = (uint16_t)v; else a.ids[idx] = v; };
	auto settle = [&](uint64_t r) -> int {
		if(r == a.v.zoff) { if(gl == 0) put(0); return R_NEED; }
		if((r & lowmask) == 0) return R_SAMPLE;
		return R_WALK;
	};
	for(;;) {
		{
			const bool want = mode == R_NEED;
			if(more) {
				unsigned long long t = 0;
				bool got = pool_take(pool, want && gl == 0, a.task_ctr, (unsigned long long)n, a.chunk, t);
				t = __shfl_sync(0xffffffffu, t, gbase); got = __shfl_sync(0xffffffffu, (int)got, gbase) != 0;
				if(want) {
					if(got) { idx = t; row = IDENT ? idx : (a.rows[idx] & kRowMask); if(COUNT && gl == 0) c_rows++; mode = settle(row); }
					else mode = R_DONE;
				}
				if(__any_sync(0xffffffffu, want && !got)) more = false;
			} else if(want) mode = R_DONE;
		}
		if(!__any_sync(0xffffffffu, mode != R_DONE)) break;
		ulonglong2 e = make_ulonglong2(0, 0); uint32_t samp = 0;
		if(mode == R_WALK && !CR) e = __ldg(r16 + r16_entry(row, (int)gl));
		else if(mode == R_SAMPLE && gl == 0) samp = a.v.sample32 ? __ldg(a.v.sample32 + (row >> a.v.off_rate)) : (uint32_t)__ldg(a.v.sample16 + (row >> a.v.off_rate));
		if(mode == R_SAMPLE) { if(gl == 0) put(samp); mode = R_NEED; }
		else if(mode == R_WALK) {
			unsigned flagged = 0;
			if(CR) { if(a.v.n_boundaries && row <= a.v.last_boundary) { const uint64_t b = row >> a.v.bshift; flagged = (a.v.bbits[b >> 5] >> (b & 31)) & 1u; } }
			else flagged = __shfl_sync(gmask, (unsigned)(e.x >> 63), gbase);     // A's entry carries the boundary flag
			bool found = false;
			if(flagged && a.v.last_boundary > 0 && row <= a.v.last_boundary) {
				uint32_t lo = 0, hi = a.v.n_boundaries;
				while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(a.v.brow[mid] < row) lo = mid + 1; else hi = mid; }
				if(lo < a.v.n_boundaries && a.v.brow[lo] == row) { found = true; if(gl == 0) put(a.v.sample32 ? a.v.bseq[lo] : (uint32_t)(uint16_t)a.v.bseq[lo]); }
			}
			if(found) mode = R_NEED;
			else {
				if(CR) row = cr_lf(a.v, row, cr_bwt(a.v, row));
				else group_lf(a.v, row, e, row);      // exactly one base owns the row: settle() took the '$' row
				if(COUNT && gl == 0) c_walk++;
				mode = settle(row);
			}
		}
	}
	if(COUNT && gl == 0 && a.ctr) { atomicAdd(&a.ctr->walk_steps, c_walk); atomicAdd(&a.ctr->rows_resolved, c_rows); }
}

// walk8: for every SA row r the state of eight successive mapLF1 steps (bt2_idx.h:2910): the bases BWT[r0..r7]
// (2 bits each, first step in the low bits) and the row reached, packed as row | bases << 40 | n_valid << 56.
// n_valid < 8 when the walk meets the '$' row.  While a search holds a single row and the next eight read
// bases equal the stored ones, eight dependent rank gathers collapse into this one 8-byte gather.
// 4 lanes per row (lane j fetches base j's rank16 entry: the 64-byte chunk is one request).
__global__ void __launch_bounds__(kSearchThreads) k_build_walk8(IndexView v, uint64_t nrows, uint64_t* out) {
	const unsigned gl = threadIdx.x & 3;
	const ulonglong2* r16 = reinterpret_cast<const ulonglong2*>(v.rank16);
	const uint64_t ngroups = (uint64_t)gridDim.x * (kSearchThreads / 4);
	const uint64_t per = (nrows + ngroups - 1) / ngroups;
	const uint64_t g = (uint64_t)blockIdx.x * (kSearchThreads / 4) + (threadIdx.x >> 2);
	// consecutive rows per group keep the first gathers of neighbouring rows in the same 64-row chunk
	for(uint64_t idx = g * per; idx < min(nrows, (g + 1) * per); idx++) {
		uint64_t row = idx, chars = 0; uint32_t nv = 0;
		for(; nv < 8; nv++) {
			if(row == v.zoff) break;
			uint64_t next;
			const int src = group_lf(v, row, __ldg(r16 + r16_entry(row, (int)gl)), next);
			if(src < 0) break;
			chars |= (uint64_t)src << (2 * nv);
			row = next;
		}
		if(gl == 0) out[idx] = (row & kWalkRowMask) | (chars << 40) | ((uint64_t)nv << 56);
	}
}

// Resolve by table: the sequence id of every SA row was precomputed at index load (k_resolve_c<.,true>), so
// resolving a row is one 2- or 4-byte gather instead of a ~8-step dependent walk.
__global__ void __launch_bounds__(256) k_lookup(const ResolveArgs a) {
	uint64_t n = *a.total; if(n > a.rows_cap) return;          // the row buffer was too small: slices have holes, the host re-runs the batch
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	for(uint64_t k = i; k < n; k += stride) { const uint64_t r = a.rows[k] & kRowMask; a.ids[k] = a.v.rtab32 ? __ldg(a.v.rtab32 + r) : (uint32_t)__ldg(a.v.rtab16 + r); }
}

// =======================================================================================
// k_compact
// =======================================================================================
// thread per unit: every lane's loads are issued together (a warp walking its units one after another measured 0.189 against
// 0.109 ms per 2 M-unit window on the bench batch)
__global__ void __launch_bounds__(128) k_compact(uint32_t n_units, const uint64_t* row_off, const uint64_t* out_off,
                                                 const OutRec* sparse, OutRec* dense, uint32_t* rec_off32, uint64_t dense_cap, unsigned int* overflow) {
	const uint32_t unit = blockIdx.x * blockDim.x + threadIdx.x;
	if(unit > n_units) return;
	if(unit == n_units) { rec_off32[unit] = (uint32_t)out_off[unit]; return; }
	const uint64_t o = out_off[unit], n = out_off[unit + 1] - o;
	rec_off32[unit] = (uint32_t)o;
	if(o + n > dense_cap) { if(n) atomicExch(overflow, 3u); return; }
	const uint64_t src = row_off[unit];
	for(uint64_t i = 0; i < n; i++) dense[o + i] = sparse[src + i];
}

// =======================================================================================
// Long units (a mate longer than kLongUnitLen bases): segmented search, join and per-unit stages (DESIGN.md section 12a).
// The batch's other units run the kernels above with the long units' flags cleared; the long units take these kernels,
// with buffers sized by their own lengths, and share the row buffer, k_lookup and the record scan with them.
// =======================================================================================
static const uint32_t kSegLen = 4096;        // bases per speculative chain (DESIGN.md section 12a)
static_assert(kLongUnitLen == CFB_LONG_UNIT_LEN && kMaxMateLen == CFB_MAX_MATE_LEN, "cf_logic.h and cfb200.h disagree on the read length limits");
struct LongTask { uint64_t hoff, soff; uint32_t unit, mate, len, nseg; };    // one searched mate: hits at hoff (2 * len slots), segments at soff (2 * nseg)
struct LongUnit { uint32_t unit, task0, ntask, pad; };
struct LongArgs {
	IndexView v; Params p; BatchView b;      // b: the batch's own flags (the short kernels see them with the long units cleared)
	const LongTask* tasks; uint32_t ntasks; const LongUnit* units; uint32_t nunits; uint64_t nsegs;
	HitRec* seg; uint32_t* sn; uint32_t* sexit;     // speculative chains
	HitRec* hits; uint32_t* nh;                     // the true lists, (task, strand) at hits + hoff + strand * len
	uint32_t* nrows; uint64_t* roff; uint32_t* hl;  // per long unit; hl: EmitRows' whole hit lengths, indexed like the row buffer
	unsigned long long* stats;                      // [0] speculative partial searches, [1] re-searched at the join
	UnitArgs u;
};
template <bool CR> struct DevStep {
	const IndexView& v; const uint8_t* fw; uint32_t len; int strand; unsigned long long n;
	__device__ void operator()(uint32_t cur, HitRec& h, uint32_t& nc, bool& done) { partial_search_dev<CR>(v, fw, len, strand, cur, h, nc, done); n++; }
};
struct ScalarStep {      // CFB_COUNT=1: the scalar search, counting the reference's operations
	const IndexView& v; const uint8_t* fw; uint32_t len; int strand; Counters* ctr;
	__device__ void operator()(uint32_t cur, HitRec& h, uint32_t& nc, bool& done) { partial_search_scalar(v, fw, len, strand, cur, h, nc, done, ctr); }
};
__device__ __forceinline__ const uint8_t* long_fw(const LongArgs& a, const LongTask& t) { return a.b.bases + (t.mate ? a.b.off[1][t.unit] : a.b.off[0][t.unit]); }
// the device flags decide which mates count (the text operator's long units are planned before their N filter is known)
__device__ __forceinline__ bool long_active(const LongArgs& a, const LongTask& t) { return ((a.b.flags[t.unit] >> t.mate) & 1u) != 0; }

// thread per (task, strand, segment): the speculative chain from the segment's first base
__global__ void __launch_bounds__(128) k_long_seg(const LongArgs a) {
	const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	unsigned long long n = 0;
	if(g < a.nsegs) {
		uint32_t lo = 0, hi = a.ntasks;          // the task holding segment g: the last with soff <= g
		while(hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if(a.tasks[mid].soff <= g) lo = mid; else hi = mid; }
		const LongTask t = a.tasks[lo];
		const uint32_t local = (uint32_t)(g - t.soff), strand = local / t.nseg, k = local - strand * t.nseg;
		const uint32_t start = k * kSegLen, stop = min(start + kSegLen, t.len);
		HitRec* out = a.seg + t.hoff + (uint64_t)strand * t.len + start;
		if(a.v.cr) { DevStep<true> step{a.v, long_fw(a, t), t.len, (int)strand, 0ull}; a.sn[g] = seg_chain(a.p, t.len, start, stop, step, out, a.sexit + g); n = step.n; }
		else { DevStep<false> step{a.v, long_fw(a, t), t.len, (int)strand, 0ull}; a.sn[g] = seg_chain(a.p, t.len, start, stop, step, out, a.sexit + g); n = step.n; }
	}
	for(int d = 16; d > 0; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
	if((threadIdx.x & 31) == 0 && n) atomicAdd(&a.stats[0], n);
}

// thread per (task, strand): the true chain from the speculative ones.  SCALAR: CFB_COUNT=1, search_strand_scalar itself.
template <bool SCALAR>
__global__ void __launch_bounds__(128) k_long_join(const LongArgs a) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= 2 * a.ntasks) return;
	const LongTask t = a.tasks[i >> 1]; const int strand = (int)(i & 1);
	HitRec* out = a.hits + t.hoff + (uint64_t)strand * t.len;
	const uint8_t* fw = long_fw(a, t);
	if(!long_active(a, t)) { a.nh[i] = 0; return; }
	if(SCALAR) {
		Counters local; memset(&local, 0, sizeof local);
		a.nh[i] = search_strand_scalar(a.v, a.p, fw, t.len, strand, out, t.len, &local);
		atomicAdd(&a.u.ctr->partial_searches, local.partial_searches); atomicAdd(&a.u.ctr->ftab_probes, local.ftab_probes);
		atomicAdd(&a.u.ctr->sides_search, local.sides_search); atomicAdd(&a.u.ctr->lf_steps, local.lf_steps);
		return;
	}
	const uint64_t s0 = t.soff + (uint64_t)strand * t.nseg;
	const HitRec* seg = a.seg + t.hoff + (uint64_t)strand * t.len;
	unsigned long long re = 0;
	if(a.v.cr) { DevStep<true> step{a.v, fw, t.len, strand, 0ull}; a.nh[i] = seg_join(a.p, t.len, kSegLen, seg, a.sn + s0, a.sexit + s0, step, out, &re); }
	else { DevStep<false> step{a.v, fw, t.len, strand, 0ull}; a.nh[i] = seg_join(a.p, t.len, kSegLen, seg, a.sn + s0, a.sexit + s0, step, out, &re); }
	if(re) atomicAdd(&a.stats[1], re);
}

// thread per task: extension, twin removal and trimming of the mate's two lists (post_search_long); the speculative chains'
// space holds the scratch
__global__ void __launch_bounds__(128) k_long_post(const LongArgs a) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= a.ntasks) return;
	const LongTask t = a.tasks[i];
	Counters local; Counters* lc = nullptr;
	if(a.u.ctr) { memset(&local, 0, sizeof local); lc = &local; }
	HitRec* F = a.hits + t.hoff; HitRec* R = F + t.len;
	post_search_long(a.v, a.p, long_fw(a, t), t.len, F, a.nh[2 * i], R, a.nh[2 * i + 1], reinterpret_cast<uint32_t*>(a.seg + t.hoff), lc);
	if(lc && local.ext_searches) {
		atomicAdd(&a.u.ctr->ext_searches, local.ext_searches); atomicAdd(&a.u.ctr->partial_searches, local.partial_searches);
		atomicAdd(&a.u.ctr->ftab_probes, local.ftab_probes); atomicAdd(&a.u.ctr->sides_search, local.sides_search); atomicAdd(&a.u.ctr->lf_steps, local.lf_steps);
	}
}

// thread per long unit: strand choice, sort, row count, a slice of the shared row buffer, rows with the scoring plan (k_prep's
// work; EMIT_ONLY after the row buffer had to grow)
template <bool EMIT_ONLY>
__global__ void __launch_bounds__(32, 1) k_long_prep(const LongArgs a) {      // the register budget of a single warp: the introsort spills below it
	const uint32_t li = blockIdx.x * blockDim.x + threadIdx.x;
	if(li >= a.nunits) return;
	const LongUnit lu = a.units[li];
	UnitHits u; u.n_mates = 0;
	for(uint32_t k = 0; k < lu.ntask; k++) {
		const uint32_t ti = lu.task0 + k; const LongTask& t = a.tasks[ti];
		if(!long_active(a, t)) continue;
		const int r = u.n_mates++;
		u.rdlen[r] = t.len;
		for(int st = 0; st < 2; st++) { u.L[r][st] = a.hits + t.hoff + (uint64_t)st * t.len; u.n[r][st] = a.nh[2 * ti + st]; }
	}
	uint64_t rows = 0;
	if(u.n_mates) {
		if(EMIT_ONLY) { CountRows cr(a.p, u); for_each_visit(a.p, u, cr); rows = cr.rows; }
		else { SortAndCount sc(a.p, u); for_each_visit(a.p, u, sc); rows = sc.rows; if(a.u.ctr) atomicAdd(&a.u.ctr->units, 1ull); }
	}
	if(rows > 0xFFFFFFFFull) rows = 0xFFFFFFFFull;
	const uint64_t off = rows ? atomicAdd(a.u.row_total, (unsigned long long)rows) : 0;
	a.nrows[li] = (uint32_t)rows; a.roff[li] = off;
	if(rows && off + rows <= a.u.rows_cap) { EmitRows er(a.p, u, a.u.rows + off, a.hl + off); for_each_visit(a.p, u, er); }
}

// thread per long unit, after k_score: hit map in the global scratch, records into the sparse buffer at the unit's rows, and
// the unit's record count and row offset for the record scan and k_compact
__global__ void __launch_bounds__(128) k_long_score(const LongArgs a) {
	const uint32_t li = blockIdx.x * blockDim.x + threadIdx.x;
	if(li >= a.nunits || *a.u.row_total > a.u.rows_cap) return;     // else the host grows the row buffer and runs the tail again
	const LongUnit lu = a.units[li];
	const uint64_t n = a.nrows[li], off = a.roff[li];
	uint32_t no = 0;
	if(n) {
		Entry* map = a.u.entries + off;
		const uint32_t nmap = score_plan<true>(a.v, a.p, a.u.rows + off, a.u.ids + off, n, map, a.hl + off);
		uint32_t mates = 0;
		for(uint32_t k = 0; k < lu.ntask; k++) mates += long_active(a, a.tasks[lu.task0 + k]) ? 1u : 0u;
		no = reduce_and_emit(a.v, a.p, mates == 2, map, nmap, a.u.tcs + off, a.u.recs_sparse + off);
	}
	a.u.nout[lu.unit] = no; a.u.row_off[lu.unit] = off;
}

// the short kernels' view of the flags: the long units' cleared
__global__ void k_mask_long(const LongUnit* units, uint32_t n, uint8_t* flags) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) flags[units[i].unit] = 0;
}

// =======================================================================================
// test hook kernels
// =======================================================================================
// LF(rows[i], chars[i]) through the scalar LF of cf_logic.h, which reads rank16 on the device; chars[i] > 3 means BWT[rows[i]]
__global__ void k_test_lf(IndexView v, const uint64_t* rows, const uint8_t* chars, uint64_t n, uint64_t* out) {
	for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const int c = chars[i] > 3 ? bwt_char(v, rows[i]) : chars[i];
		out[i] = lf_scalar(v, rows[i], c);
	}
}

// =======================================================================================
// host side: index replica, contexts, batches
// =======================================================================================
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
	va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap); return code;
}
#define CK(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) return fail(CFB_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while(0)

extern "C" const char* cfb_last_error(void) { return g_err; }
int cfb_fail_msg(int code, const char* msg) { return fail(code, "%s", msg); }      // for the other translation units (cf_gunzip.cu)
extern "C" const char* cfb_version(void) { return "cfb200 0.1 (sm_90a)"; }

struct cfb_index {
	HostIndex h;
	int device = -1;
	IndexView view;            // device pointers (taxonomy-independent part)
	std::vector<DBuf<uint8_t>> dptrs;
	uint64_t device_bytes = 0;
	int sm_count = 0;
	cfb_index_tables tables;
	cfb_index() { memset(&tables, 0, sizeof tables); }
	~cfb_index() { if(!dptrs.empty()) cudaSetDevice(device); }
	// a device array of the replica: `bytes` allocated, `counted` of them reported in device_bytes
	template <class T> cudaError_t alloc(size_t bytes, uint64_t counted, T** out) {
		DBuf<uint8_t> b;
		const cudaError_t e = b.alloc(bytes);
		if(e != cudaSuccess) return e;
		*out = (T*)b.p; dptrs.push_back(std::move(b)); device_bytes += counted;
		return cudaSuccess;
	}
};

static int upload(cfb_index* ix, const void* src, size_t bytes, const void** dst) {
	void* d = nullptr;
	CK(ix->alloc(bytes ? bytes : 16, bytes, &d));
	if(bytes) CK(cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice));
	*dst = d;
	return CFB_OK;
}

// file[off, off+bytes) -> device memory through a ring of pinned buffers: parallel preads fill one buffer while
// the previous one is on its way over PCIe.  No host copy of the array is kept.
static int stream_to_device(cfb_index* ix, const std::string& path, uint64_t off, uint64_t bytes, const void** dst) {
	void* d = nullptr;
	CK(ix->alloc(bytes + 64, bytes, &d));
	*dst = d;
	if(bytes == 0) return CFB_OK;
	const int fd = open(path.c_str(), O_RDONLY);
	if(fd < 0) return fail(CFB_EIO, "could not open %s", path.c_str());
	const size_t kBuf = 64u << 20; const int kRing = 3, kThreads = 8;
	HBuf<uint8_t> hb[kRing]; Event ev[kRing]; Stream st;
	int rc = CFB_OK;
	for(int i = 0; i < kRing; i++) { if(hb[i].alloc(kBuf) != cudaSuccess || ev[i].create(cudaEventDisableTiming) != cudaSuccess) rc = fail(CFB_ENOMEM, "pinned staging buffers"); }
	if(rc == CFB_OK && st.create() != cudaSuccess) rc = fail(CFB_ECUDA, "stream");
	uint64_t done = 0; int k = 0;
	while(rc == CFB_OK && done < bytes) {
		const size_t n = (size_t)std::min<uint64_t>(kBuf, bytes - done);
		const int b = k % kRing;
		if(k >= kRing && cudaEventSynchronize(ev[b]) != cudaSuccess) { rc = fail(CFB_ECUDA, "event"); break; }
		std::atomic<bool> bad(false);
		auto piece = [&](int t) {
			const size_t lo = n * t / kThreads, hi = n * (t + 1) / kThreads; size_t got = lo;
			while(got < hi) { const ssize_t r = pread(fd, hb[b].p + got, hi - got, (off_t)(off + done + got)); if(r <= 0) { bad = true; return; } got += (size_t)r; }
		};
		std::vector<std::thread> th;
		for(int t = 1; t < kThreads; t++) th.emplace_back(piece, t);
		piece(0);
		for(size_t t = 0; t < th.size(); t++) th[t].join();
		if(bad) { rc = fail(CFB_EIO, "short read in %s", path.c_str()); break; }
		if(cudaMemcpyAsync((uint8_t*)d + done, hb[b].p, n, cudaMemcpyHostToDevice, st) != cudaSuccess || cudaEventRecord(ev[b], st) != cudaSuccess) { rc = fail(CFB_ECUDA, "H2D of %s", path.c_str()); break; }
		done += n; k++;
	}
	if(st && cudaStreamSynchronize(st) != cudaSuccess && rc == CFB_OK) rc = fail(CFB_ECUDA, "H2D of %s", path.c_str());
	close(fd);
	return rc;
}

extern "C" int cfb_index_load_ex(const char* basename, int device, uint32_t flags, cfb_index** out) {
	if(!basename || !out) return fail(CFB_EINVAL, "cfb_index_load: null argument");
	std::unique_ptr<cfb_index> ix(new cfb_index());       // the half-built replica goes with every error return
	std::string err = load_cf_index(basename, ix->h, /*defer_bulk=*/device >= 0);
	if(!err.empty()) return fail(CFB_EIO, "%s", err.c_str());
	const HostIndex& h = ix->h;
	ix->device = device;
	if(device >= 0) {
		if(h.line_rate != 7) return fail(CFB_EFORMAT, "index lineRate %d unsupported: the kernels require 128-byte sides (centrifuge-build default --linerate 7)", h.line_rate);
		if(h.ftab_chars > 15) return fail(CFB_EFORMAT, "ftabChars %d unsupported", h.ftab_chars);
		int ndev = 0;
		if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) return fail(CFB_ENODEV, "no CUDA device %d (found %d); this library has no CPU fallback", device, ndev);
		cudaDeviceProp prop;
		if(cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(CFB_ENODEV, "cannot use CUDA device %d", device);
		ix->sm_count = prop.multiProcessorCount;
		IndexView& v = ix->view; memset(&v, 0, sizeof v);
		int rc;
		// The rank layout, chosen before anything is allocated (choose_rank_layout): rank16 (1 byte per row, built beside the
		// streamed sides, which it replaces) when it fits with everything else, else the compact layout (1/3 byte per row, built in
		// place from the sides).  Head-room as for the derived tables below.  CFB_RANK16=0 forces the compact layout (tests, A/B).
		size_t free0 = 0, total0 = 0; cudaMemGetInfo(&free0, &total0);
		double head_gb = 12.0; { const char* e = getenv("CFB_HBM_HEADROOM_GB"); if(e) head_gb = atof(e); }
		const uint64_t headroom0 = std::min<uint64_t>((uint64_t)(head_gb * 1073741824.0), free0 / 2);
		const uint64_t sample_b = h.offs_len * (h.wide_sample ? 4 : 2);
		const uint64_t fixed_b = (h.ftab.size() + h.eftab.size() + h.brow.size() + h.seq_taxid.size() + h.paths.size()) * 8
		                       + (h.bseq.size() + h.bbits.size() + h.seq_path.size()) * 4 + (h.ftab_len - 1) * 16 + cr_superblocks(h.num_sides) * 32;
		const char* er = getenv("CFB_RANK16");
		const int layout = choose_rank_layout(free0, h.num_sides, sample_b, fixed_b, headroom0, er && er[0] == '0');
		if(layout == kLayoutNone) {
			const unsigned long long nr = rank16_bytes_for(h.num_sides) + h.num_sides * 128, nc = cr_bytes_for(h.num_sides), rest = sample_b + fixed_b + headroom0;
			return fail(CFB_ENOMEM, "index %s fits no rank layout on device %d: rank16 needs %llu bytes and the compact layout %llu, each plus %llu bytes "
			            "of sample, fixed tables and head-room; %llu bytes are free", basename, device, nr + rest, nc + rest, rest, (unsigned long long)free0);
		}
		auto up = [&](const auto& vec, auto*& field) { return upload(ix.get(), vec.data(), vec.size() * sizeof(vec[0]), (const void**)&field); };
		ix->tables.sample_bytes = h.offs_len * (h.wide_sample ? 4 : 2);
		if((rc = stream_to_device(ix.get(), std::string(basename) + ".1.cf", h.sides_file_off, h.num_sides * h.side_sz, (const void**)&v.sides)) ||
		   (rc = up(h.ftab, v.ftab)) || (rc = up(h.eftab, v.eftab)) ||
		   (rc = stream_to_device(ix.get(), std::string(basename) + ".2.cf", h.sample_file_off, h.offs_len * (h.wide_sample ? 4 : 2),
		                          h.wide_sample ? (const void**)&v.sample32 : (const void**)&v.sample16)) ||
		   (rc = up(h.brow, v.brow)) || (rc = up(h.bseq, v.bseq)) || (rc = up(h.bbits, v.bbits)) ||
		   (rc = up(h.seq_taxid, v.seq_taxid)) || (rc = up(h.seq_path, v.seq_path)) || (rc = up(h.paths, v.paths))) return rc;
		v.len = h.len; v.zoff = h.zoff; v.zside = h.zoff / 384; v.zoffc = (uint32_t)(h.zoff % 384);
		for(int i = 0; i < 4; i++) v.fchr[i] = h.fchr[i];
		v.last_boundary = h.last_boundary; v.num_sides = h.num_sides;
		v.n_boundaries = (uint32_t)h.brow.size(); v.n_seqs = (uint32_t)h.seq_taxid.size();
		v.off_rate = h.off_rate; v.ftab_chars = h.ftab_chars; v.bshift = h.bshift;
		{   // 16-byte rank entries + fused ftab for the walk kernels
			const bool compact = layout == kLayoutCompact;
			uint64_t* r16 = nullptr; const uint64_t nb = h.num_sides * 6;
			if(compact) {
				const uint64_t nsb = cr_superblocks(h.num_sides);
				uint64_t* sb = nullptr;
				CK(ix->alloc(nsb * 32, nsb * 32, &sb));
				k_cr_superblocks<<<(unsigned)((nsb + 255) / 256), 256>>>(v.sides, h.num_sides, h.zoff, nsb, sb);
				k_cr_convert<<<(unsigned)((h.num_sides + 255) / 256), 256>>>(const_cast<uint64_t*>(v.sides), h.num_sides, h.zoff, sb);
				v.crsb = sb;
			} else {
				CK(ix->alloc((nb + 1) * 64, (nb + 1) * 64, &r16));
				k_build_rank16<<<(unsigned)((nb + 1 + 255) / 256), 256>>>(v.sides, h.num_sides, v.zside, v.zoffc, r16);
				if(v.n_boundaries) k_mark_boundaries<<<(v.n_boundaries + 255) / 256, 256>>>(v.brow, v.n_boundaries, r16);
			}
			uint64_t* f2 = nullptr; const uint64_t nf = h.ftab_len - 1;
			CK(ix->alloc(nf * 16, nf * 16, &f2));
			k_build_ftab2<<<(unsigned)((nf + 255) / 256), 256>>>(v, nf, f2);
			CK(cudaDeviceSynchronize());
			v.ftab2 = f2; ix->tables.ftab2_bytes = nf * 16;
			if(compact) {      // the converted sides are the rank structure: sides_bytes reports them
				v.cr = v.sides; v.sides = nullptr;
				ix->tables.sides_bytes = cr_bytes_for(h.num_sides);
			} else {
				v.rank16 = r16;
				ix->tables.rank16_bytes = (nb + 1) * 64;
				// The file's sides were only the staging buffer of rank16, which holds the same information (the scalar LF of the
				// extension step reads rank16 too): no kernel reads them from here on.
				ix->dptrs.erase(std::find_if(ix->dptrs.begin(), ix->dptrs.end(), [&](const DBuf<uint8_t>& b) { return (const void*)b.p == (const void*)v.sides; }));
				ix->device_bytes -= h.num_sides * h.side_sz; v.sides = nullptr;
			}
			// HBM budget of the derived tables: what is free now minus the head-room the batch buffers need (12 GB by default, 15 % of an
			// 80 GB H100: 4 slots of 0.5 M 100 bp reads in flight at ~3 KB each with 30 % to grow,
			// plus 3 GB of fixed buffers; callers that keep more in flight set CFB_HBM_HEADROOM_GB, as bench.py does).  Tables are built in the order of gathers saved per
			// byte -- K-mer jump table, resolve table, walk8 -- each only if it fits what is left; walk8, whose rows are hit
			// uniformly, may cover just a prefix of the rows (a jump needs the entries of the range's two end rows only).  With
			// range jumps, K = 14 (4.3 GB, walk8 on 34 % of the bench index's rows instead of 16 %) measured the same as K = 15
			// (274.5 vs 274.6-275.7 M reads/s on one H100 80GB HBM3 at 400 W), so the K-mer table keeps its place in the order.
			size_t free_b = 0, total_b = 0; cudaMemGetInfo(&free_b, &total_b);
			const uint64_t headroom = std::min<uint64_t>((uint64_t)(head_gb * 1073741824.0), free_b / 2);
			auto budget = [&]() -> uint64_t { size_t f = 0, t = 0; cudaMemGetInfo(&f, &t); return f > headroom ? f - headroom : 0; };
			// K-mer jump table with its death bitmap: K = largest value with 4^K <= len/4 (most K-mers occur), capped at 15 and by
			// the budget.  Where no K above ftabChars fits (small indexes, CFB_FTABK=10) it is still built at K = ftabChars
			// (16 MB) for the bitmap alone, unless that is switched off too (CFB_FTABD=0).
			{
				const char* ed = getenv("CFB_FTABD");
				const bool death = !(ed && ed[0] == '0');
				int K = 0;
				{ const char* e = getenv("CFB_FTABK"); if(e) K = atoi(e); else { K = h.ftab_chars; while(K < 15 && (4ull << (2 * K)) <= h.len / 4) K++; } }
				while(K > h.ftab_chars && (16ull << (2 * K)) > budget() / 2) K--;
				if(K <= h.ftab_chars || K > 16) K = death ? h.ftab_chars : 0;
				const uint64_t nk = K ? 1ull << (2 * K) : 0;
				if(K && h.len + 1 < (1ull << 40) && nk * 16 <= budget()) {
					ulonglong2* fk = nullptr;
					CK(ix->alloc(nk * 16, nk * 16, &fk));
					k_build_ftabk<<<(unsigned)((nk + 127) / 128), 128>>>(v, K, nk, death, fk);
					CK(cudaDeviceSynchronize());
					v.ftabk = (const uint64_t*)fk; v.ftabk_chars = K; v.ftabd_chars = death ? K + 3 : 0;
					ix->tables.ftabk_bytes = nk * 16; ix->tables.ftabk_chars = K; ix->tables.ftabd_chars = v.ftabd_chars;
				}
			}
			// resolve table: sequence id of every SA row (walked once here).  Neither it nor walk8 is built on the compact layout: at the
			// sizes that need it they would not fit, and they never change results.
			if(!compact) {
				const char* e = (flags & CFB_LOAD_NO_RESOLVE_TABLE) ? "0" : getenv("CFB_RESOLVE_TABLE");
				const uint64_t nrows = h.len + 1, esz = h.wide_sample ? 4 : 2;
				if(!(e && e[0] == '0') && nrows * esz + 16 <= budget()) {
					void* tab = nullptr; DBuf<unsigned long long> sc;
					CK(ix->alloc(nrows * esz + 16, nrows * esz, &tab)); CK(sc.alloc(2));
					const unsigned long long init[2] = {0ull, (unsigned long long)nrows};
					CK(cudaMemcpy(sc.p, init, 16, cudaMemcpyHostToDevice));
					ResolveArgs ra; ra.v = v; ra.rows = nullptr; ra.ids = h.wide_sample ? (uint32_t*)tab : nullptr; ra.ids16 = h.wide_sample ? nullptr : (uint16_t*)tab;
					ra.total = (const uint64_t*)(sc.p + 1); ra.rows_cap = nrows; ra.task_ctr = sc.p; ra.chunk = 256; ra.ctr = nullptr;
					int occ = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_resolve_c<false, true>, kSearchThreads, 0);
					k_resolve_c<false, true><<<prop.multiProcessorCount * std::max(occ, 1), kSearchThreads>>>(ra);
					CK(cudaDeviceSynchronize());
					if(h.wide_sample) v.rtab32 = (const uint32_t*)tab; else v.rtab16 = (const uint16_t*)tab;
					ix->tables.resolve_table_bytes = nrows * esz; ix->tables.resolve_entry_bytes = (int32_t)esz;
				}
			}
			// walk8: eight single-row LF steps per gather, for as many rows as the budget allows (at least an eighth of them)
			if(!compact) {
				const char* e = (flags & CFB_LOAD_NO_WALK8) ? "0" : getenv("CFB_WALK8");
				const uint64_t nrows = h.len + 1;
				uint64_t cover = std::min<uint64_t>(nrows, budget() / 8);
				{ const char* f = getenv("CFB_WALK8_ROWS"); if(f) cover = std::min<uint64_t>(nrows, strtoull(f, NULL, 10)); }     // tests: force a partial table
				if(!(e && e[0] == '0') && nrows < (1ull << 40) && cover >= nrows / 8 && cover > 0) {
					void* tab = nullptr;
					CK(ix->alloc(cover * 8 + 16, cover * 8, &tab));
					int occ = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_build_walk8, kSearchThreads, 0);
					k_build_walk8<<<prop.multiProcessorCount * std::max(occ, 1) * 4, kSearchThreads>>>(v, cover, (uint64_t*)tab);
					CK(cudaDeviceSynchronize());
					v.walk8 = (const uint64_t*)tab; v.walk8_rows = cover;
					ix->tables.walk8_bytes = cover * 8; ix->tables.walk8_rows = cover;
				}
			}
		}
		{ size_t fb = 0, tb = 0; cudaMemGetInfo(&fb, &tb); ix->tables.total_bytes = ix->device_bytes; ix->tables.free_bytes_after_load = fb; }
		// host copies of the big arrays are no longer needed once uploaded
		std::vector<uint8_t>().swap(ix->h.sides);
	}
	*out = ix.release();
	return CFB_OK;
}
extern "C" int cfb_index_load(const char* basename, int device, cfb_index** out) { return cfb_index_load_ex(basename, device, 0u, out); }
extern "C" void cfb_index_free(cfb_index* ix) { delete ix; }
extern "C" int cfb_index_get_info(const cfb_index* ix, cfb_index_info* o) {
	if(!ix || !o) return fail(CFB_EINVAL, "null argument");
	const HostIndex& h = ix->h;
	o->len = h.len; o->num_sides = h.num_sides; o->n_seqs = h.seq_taxid.size(); o->n_tax_nodes = h.nodes.size();
	o->n_boundaries = h.brow.size(); o->line_rate = h.line_rate; o->off_rate = h.off_rate; o->ftab_chars = h.ftab_chars;
	o->sample_bytes = h.wide_sample ? 4 : 2; o->compressed = h.compressed ? 1 : 0; o->device = ix->device; o->device_bytes = ix->device_bytes;
	return CFB_OK;
}
extern "C" int cfb_index_get_tables(const cfb_index* ix, cfb_index_tables* o) {
	if(!ix || !o) return fail(CFB_EINVAL, "null argument");
	*o = ix->tables;
	return CFB_OK;
}
extern "C" const char* cfb_index_seq_name(const cfb_index* ix, uint32_t s) { return (ix && s < ix->h.seq_name.size()) ? ix->h.seq_name[s].c_str() : NULL; }
extern "C" uint64_t cfb_index_seq_taxid(const cfb_index* ix, uint32_t s) { return (ix && s < ix->h.seq_taxid.size()) ? ix->h.seq_taxid[s] : 0; }
extern "C" int cfb_index_tax_node(const cfb_index* ix, uint64_t taxid, uint64_t* parent, int* rank, int* leaf) {
	const TaxNode* n = ix ? ix->h.find_node(taxid) : NULL;
	if(!n) return 0;
	if(parent) *parent = n->parent; if(rank) *rank = n->rank; if(leaf) *leaf = n->leaf;
	return 1;
}
// internal accessor for the host driver (cf_host.cpp); not part of the public C ABI
extern "C" const cfb::HostIndex* cfb_index_host(const cfb_index* ix) { return ix ? &ix->h : NULL; }
extern "C" int cfb_index_node_taxids(const cfb_index* ix, uint64_t* out, uint64_t cap) {
	if(!ix || !out || cap < ix->h.nodes.size()) return fail(CFB_EINVAL, "cfb_index_node_taxids: buffer too small");
	for(size_t i = 0; i < ix->h.nodes.size(); i++) out[i] = ix->h.nodes[i].taxid;
	return CFB_OK;
}
extern "C" void cfb_params_default(cfb_params* p) {
	if(!p) return;
	memset(p, 0, sizeof *p); p->khits = 5; p->min_hitlen = 22; p->tree_traverse = 1; p->class_rank_slot = 0;
}

// ---------------------------------------------------------------------------------------
static const int kSlots = 17;  // 16 pipelined slots (two waves of 8 sub-batches keep the copy engines busy across batch boundaries) + 1 for resident batches

struct Slot {
	Stream st; Event ev[6];
	// inputs
	HBuf<uint8_t> h_bases; HBuf<uint64_t> h_off; HBuf<uint32_t> h_len; HBuf<uint8_t> h_flags;
	DBuf<uint8_t> d_bases; DBuf<uint64_t> d_off; DBuf<uint32_t> d_len; DBuf<uint8_t> d_flags;
	HBuf<uint64_t> h_words; DBuf<uint64_t> d_words, d_npos, d_woff; DBuf<uint32_t> d_wlen;      // packed input (cfb_batch_packed)
	// work
	DBuf<uint64_t> pk; DBuf<uint32_t> nm;
	DBuf<HitRec> hits; DBuf<uint32_t> nhits; DBuf<HitRec> regen; DBuf<uint32_t> regen_n; uint64_t regen_slots = 0; uint32_t full_cap = 0; DBuf<uint32_t> nrows; DBuf<uint64_t> row_off; DBuf<uint64_t> bsum;
	DBuf<uint64_t> rows; DBuf<uint32_t> ids; DBuf<Entry> entries; DBuf<TaxCnt> tcs; DBuf<OutRec> sparse;
	DBuf<uint32_t> nout; DBuf<uint64_t> out_off; DBuf<uint8_t> scan_tmp; DBuf<OutRec> dense; DBuf<uint32_t> rec_off32;
	DBuf<unsigned long long> scal;    // [0] search task ctr (u32 used), [1] resolve ctr, [2] overflow, [3] total rows, [4] total recs
	HBuf<unsigned long long> h_scal;
	HBuf<OutRec> h_recs; HBuf<uint32_t> h_rec_off;
	DBuf<unsigned long long> cnt;     // this batch's per-taxon counters (record path), added to the context's totals at wait time
	bool folded = false, is_text = false, commit_pending = false;
	NCeil nceil; bool custom_nceil = false;   // the batch's N ceiling when it is not the default: sizes the hit lists (nceil_full_cap)
	// batch bookkeeping
	BatchView bv; uint64_t n_units = 0, n_bases = 0; uint32_t maxlen = 0, cap = 0; uint64_t rows_cap = 0, dense_cap = 0;
	bool pending = false, reran = false;
	bool want_host = false; uint64_t d2h_recs = 0;     // records already copied to h_recs by the speculative D2H queued behind the kernels
	// long units of the staged batch (absolute unit index, mate lengths, flags) and the window the kernels run (resident ranges)
	struct LongH { uint64_t unit; uint32_t len[2]; uint8_t fl; };
	std::vector<LongH> longs; uint64_t win_first = 0; uint32_t nlong_win = 0;
	HBuf<LongTask> h_ltask; HBuf<LongUnit> h_lunit; DBuf<LongTask> d_ltask; DBuf<LongUnit> d_lunit;
	DBuf<HitRec> lseg, lhits; DBuf<uint32_t> lsn, lsexit, lnh, lnrows, lhl; DBuf<uint64_t> lroff; DBuf<uint8_t> flags_short; DBuf<unsigned long long> lstats;
	uint64_t lhit_slots = 0, lsegs = 0; uint32_t lntasks = 0, lmaxlen = 0;
};

struct cfb_dbatch { int slot; uint64_t n_units; };
struct TextCtx;                       // cf_text.cuh

// Per-taxon counters of a context, on the device (SpeciesMetrics::addSpeciesCounts, aln_sink.h:142-172): for every taxid
// the report can mention -- tree nodes, sequence taxids, 0 and 1 -- {numReads, numUniqueReads, reads whose single
// best row reached the maximum score}.  Both the text operator (k_fmt_plan) and the record-level path (k_fold_counts,
// when cfb_ctx_count_records is on) add to `total` when a batch is collected; cfb_counts_allreduce sums `total` over the
// communicator's ranks into `global` (NCCL, ncclUint64, ncclSum).
struct CountsCtx {
	bool ready = false;
	std::vector<uint64_t> h_taxid; DBuf<uint64_t> d_taxid; uint32_t n = 0;
	DBuf<unsigned long long> total, global; bool reduced = false;
};

struct cfb_ctx {
	const cfb_index* ix = nullptr;
	IndexView view; Params prm;
	DBuf<uint64_t> d_host; DBuf<SeqInfo> d_seqs;
	Slot slots[kSlots];
	DBuf<Counters> d_ctr; int count = 0;        // CFB_COUNT: 1 = reference operation counters, 2 = the product's own load requests
	uint64_t launches = 0;
	int resolve_blocks = 0;
	cfb_dbatch resident; bool resident_used = false;
	double rec_ratio = 2.0;       // records per unit seen so far (sizes the speculative D2H)
	uint64_t rows_cap0 = 0;       // CFB_ROWS_CAP: initial row-buffer capacity (tests force the grow-and-re-run path with it)
	std::unique_ptr<TextCtx> text;
	NCeil nceil;                  // cfb_ctx_set_n_ceil: the text operator's N filter, and the hit-list bound of every later batch
	Quals quals;                  // cfb_ctx_set_quals: the quality encoding of later text spans
	CountsCtx cnt; bool fold_records = false;
	bool keep_short = false;      // CFB_KEEP_SHORT=1: store every hit (A/B and tests)
	uint64_t long_units = 0, long_bases = 0, long_searches = 0, long_researched = 0;    // cfb_ctx_long_stats
	uint64_t regen_lists = 0, regen_tasks = 0;   // lists regenerated / strand lists searched so far (CFB_REGEN_STATS=1 prints them when the context goes)
	uint64_t regen_slots0 = 0;    // CFB_REGEN_SLOTS: initial capacity of the list-regeneration buffer (tests force the grow-and-re-run path with it)
	void* comm = nullptr; int comm_rank = 0, comm_size = 1; Stream comm_st;      // NCCL communicator (cf_multi.cuh)
	~cfb_ctx();       // after cf_multi.cuh, where TextCtx is complete
};

// every tree node whose ancestor chain contains a listed id (Classifier ctor classifier.h:157-201)
static void expand_taxids(const HostIndex& h, const uint64_t* ids, uint64_t n, std::set<uint64_t>& out) {
	if(n == 0 || !ids) return;
	for(size_t i = 0; i < h.nodes.size(); i++) {
		uint64_t t = h.nodes[i].taxid;
		for(;;) {
			bool found = false;
			for(uint64_t k = 0; k < n; k++) if(ids[k] == t) { found = true; break; }
			if(found) { out.insert(h.nodes[i].taxid); break; }
			const TaxNode* nd = h.find_node(t);
			if(!nd || nd->parent == t) break;
			t = nd->parent;
		}
	}
}

extern "C" void cfb_ctx_destroy(cfb_ctx* c) { delete c; }

extern "C" int cfb_ctx_create(const cfb_index* ix, const cfb_params* p, cfb_ctx** out) {
	if(!ix || !p || !out) return fail(CFB_EINVAL, "cfb_ctx_create: null argument");
	if(ix->device < 0) return fail(CFB_ENODEV, "index was loaded host-only; classification needs a CUDA device (no CPU fallback)");
	if(p->khits < 1) return fail(CFB_EINVAL, "khits must be >= 1");
	CK(cudaSetDevice(ix->device));
	std::unique_ptr<cfb_ctx> c(new cfb_ctx());        // the half-built context goes with every error return
	c->ix = ix; c->view = ix->view;
	const HostIndex& h = ix->h;
	Params& q = c->prm;
	q.khits = (uint32_t)p->khits;
	q.min_hitlen = (uint32_t)(p->min_hitlen < 15 ? 15 : p->min_hitlen);
	q.ihits = (uint32_t)std::max(p->khits, 5) * (h.compressed ? 4u : 40u);       // ReportingParams aln_sink.h:580-588
	q.increment = (2 * q.min_hitlen <= 33) ? 10 : (2 * q.min_hitlen - 33);        // classifier.h:226
	q.tree_traverse = p->tree_traverse ? 1 : 0;
	q.class_rank_slot = (uint32_t)(p->class_rank_slot & 0xff);
	std::set<uint64_t> host, excl;
	expand_taxids(h, p->host_taxids, p->n_host_taxids, host);
	expand_taxids(h, p->excluded_taxids, p->n_excluded_taxids, excl);
	// the exclude set reaches the device only through the sequence table: seq_info_of reads the flags for ids < n_seqs alone
	std::vector<uint8_t> fl;
	if(!excl.empty()) {
		fl.assign(h.seq_taxid.size(), 0);
		for(size_t i = 0; i < fl.size(); i++) fl[i] = excl.count(h.seq_taxid[i]) ? 1 : 0;
	}
	{     // seq_info_of every sequence id under this context's rank and exclude set: k_score reads one 16-byte record per distinct id
		IndexView hv; memset(&hv, 0, sizeof hv);
		hv.seq_taxid = h.seq_taxid.data(); hv.seq_path = h.seq_path.data(); hv.paths = h.paths.data(); hv.n_seqs = (uint32_t)h.seq_taxid.size();
		hv.seq_excluded = fl.empty() ? nullptr : fl.data();
		std::vector<SeqInfo> tab(hv.n_seqs);
		for(uint32_t i = 0; i < hv.n_seqs; i++) tab[i] = seq_info_of(hv, q, i);
		CK(c->d_seqs.ensure(tab.size() + 1)); CK(cudaMemcpy(c->d_seqs.p, tab.data(), tab.size() * sizeof(SeqInfo), cudaMemcpyHostToDevice));
		c->view.seqs = c->d_seqs.p;
	}
	if(!host.empty()) {
		std::vector<uint64_t> hv(host.begin(), host.end());
		CK(c->d_host.ensure(hv.size())); CK(cudaMemcpy(c->d_host.p, hv.data(), hv.size() * 8, cudaMemcpyHostToDevice));
		c->view.host_taxids = c->d_host.p; c->view.n_host = (uint32_t)hv.size();
	}
	for(int i = 0; i < kSlots; i++) {
		CK(c->slots[i].st.create());
		for(int e = 0; e < 6; e++) CK(c->slots[i].ev[e].create());
		CK(c->slots[i].scal.ensure(8)); CK(c->slots[i].h_scal.ensure(8));
	}
	CK(c->d_ctr.alloc(1)); CK(cudaMemset(c->d_ctr.p, 0, sizeof(Counters)));
	// random 32-byte sector gathers: do not let L2 over-fetch neighbouring sectors from HBM
	cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
	cudaGetLastError();
	int occ = 0;
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_resolve_c<false, false>, kSearchThreads, 0));
	c->resolve_blocks = ix->sm_count * std::max(occ, 1);
	{ const char* rc0 = getenv("CFB_ROWS_CAP"); if(rc0) c->rows_cap0 = strtoull(rc0, NULL, 10); }
	{ const char* ks = getenv("CFB_KEEP_SHORT"); c->keep_short = ks && ks[0] == '1'; }
	{ const char* rs = getenv("CFB_REGEN_SLOTS"); if(rs) c->regen_slots0 = strtoull(rs, NULL, 10); }
	const char* cnt = getenv("CFB_COUNT");
	c->count = cnt ? (cnt[0] == '1' ? 1 : (cnt[0] == '2' ? 2 : 0)) : 0;
	*out = c.release();
	return CFB_OK;
}
extern "C" int cfb_ctx_slots(const cfb_ctx*) { return kSlots - 1; }   // last slot is reserved for resident batches
extern "C" int cfb_ctx_kernel_launches(const cfb_ctx* c, uint64_t* n) { if(!c || !n) return CFB_EINVAL; *n = c->launches; return CFB_OK; }

// ---------------------------------------------------------------------------------------
// per-taxon counters of the record-level path
// ---------------------------------------------------------------------------------------
static int counts_init(cfb_ctx* c) {
	CountsCtx& k = c->cnt;
	if(k.ready) return CFB_OK;
	const HostIndex& h = c->ix->h;
	std::set<uint64_t> sp; sp.insert(0); sp.insert(1);
	for(size_t i = 0; i < h.nodes.size(); i++) sp.insert(h.nodes[i].taxid);
	sp.insert(h.seq_taxid.begin(), h.seq_taxid.end());
	k.h_taxid.assign(sp.begin(), sp.end()); k.n = (uint32_t)k.h_taxid.size();
	CK(k.d_taxid.ensure(k.n + 1)); CK(cudaMemcpy(k.d_taxid.p, k.h_taxid.data(), (size_t)k.n * 8, cudaMemcpyHostToDevice));
	CK(k.total.ensure(3ull * k.n)); CK(cudaMemset(k.total.p, 0, 3ull * k.n * 8));
	CK(k.global.ensure(3ull * k.n)); CK(cudaMemset(k.global.p, 0, 3ull * k.n * 8));
	k.ready = true;
	return CFB_OK;
}

struct FoldArgs {
	const uint64_t* sp_taxid; uint32_t n_sp;
	const uint32_t* rec_off; const OutRec* recs; uint32_t n_units; int32_t n_mates; uint32_t khits;
	const uint32_t* len[2]; const uint8_t* flags;
	unsigned long long* sp;        // 3 * n_sp: numReads | numUniqueReads | observed singletons
};
__device__ __forceinline__ int find_slot(const uint64_t* a, uint32_t n, uint64_t key) {
	uint32_t lo = 0, hi = n;
	while(lo < hi) { const uint32_t mid = (lo + hi) >> 1; if(a[mid] < key) lo = mid + 1; else hi = mid; }
	return (lo < n && a[lo] == key) ? (int)lo : -1;
}
// thread per unit: what AlnSinkWrap::finishRead -> SpeciesMetrics::addSpeciesCounts accumulate for the unit's reported
// assignments (aln_sink.h:142-172,1861-1927): the records with the best score, at most khits of them (hit-map order; a tie
// of more than khits records is resolved by the per-read RNG in the reference and in the text operator -- it only arises
// under --host-taxids).  A unit without records counts as taxid 0, as its "unclassified" row does.
__global__ void __launch_bounds__(128) k_fold_counts(const FoldArgs a) {
	const uint32_t u = blockIdx.x * 128 + threadIdx.x;
	const bool live = u < a.n_units;
	int first_slot = -1; uint32_t num = 1; bool qualifies = false;
	if(live) {
		const uint32_t r0 = a.rec_off[u], r1 = a.rec_off[u + 1];
		if(r1 == r0) { first_slot = find_slot(a.sp_taxid, a.n_sp, 0); qualifies = true; }
		else {
			uint32_t best = 0, ties = 0;
			for(uint32_t k = r0; k < r1; k++) { const uint32_t sc = a.recs[k].score; if(sc > best || k == r0) { best = sc; ties = 1; } else if(sc == best) ties++; }
			num = ties < a.khits ? ties : a.khits;
			const uint32_t fl = a.flags ? a.flags[u] : 3u;
			int64_t max_score = 0;
			if(fl & 1u) { const int64_t L = a.len[0][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
			if(a.n_mates == 2 && (fl & 2u)) { const int64_t L = a.len[1][u]; max_score += L > 15 ? (L - 15) * (L - 15) : 0; }
			qualifies = (int64_t)best >= max_score;
			uint32_t taken = 0;
			for(uint32_t k = r0; k < r1 && taken < num; k++) {
				if(a.recs[k].score != best) continue;
				const int slot = find_slot(a.sp_taxid, a.n_sp, a.recs[k].taxid);
				if(taken == 0) first_slot = slot; else if(slot >= 0) atomicAdd(a.sp + slot, 1ull);
				taken++;
			}
		}
	}
	// first assignment of every unit: warp-aggregated (dominant taxa would serialise per-lane atomics)
	const int key = live ? first_slot : -1;
	const uint32_t peers = __match_any_sync(0xffffffffu, key);
	if(key >= 0) {
		const uint32_t uniq = __popc(__ballot_sync(peers, num == 1) & peers);
		const uint32_t obs = __popc(__ballot_sync(peers, num == 1 && qualifies) & peers);
		if((uint32_t)(__ffs(peers) - 1) == (threadIdx.x & 31u)) {
			atomicAdd(a.sp + key, (unsigned long long)__popc(peers));
			if(uniq) atomicAdd(a.sp + a.n_sp + key, (unsigned long long)uniq);
			if(obs) atomicAdd(a.sp + 2ull * a.n_sp + key, (unsigned long long)obs);
		}
	}
}
__global__ void k_cnt_commit(const unsigned long long* slot_sp, unsigned long long* total, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) { const unsigned long long v = slot_sp[i]; if(v) atomicAdd(total + i, v); }
}

// Validate + stage a batch into the slot's pinned buffers and enqueue H2D copies.
// Device memory a batch with long units could not get: CFB_ENOMEM naming the long reads (other batches report CFB_ECUDA as before)
static int long_oom(const Slot& s, cudaError_t e, const char* what) {
	cudaGetLastError();
	uint64_t bases = 0; uint32_t mx = 0;
	for(const Slot::LongH& l : s.longs) { bases += (uint64_t)l.len[0] + l.len[1]; mx = std::max(mx, std::max(l.len[0], l.len[1])); }
	return fail(CFB_ENOMEM, "no device memory for %s of a batch with %zu long units (%llu bases, the longest read %u bases): %s", what,
	            s.longs.size(), (unsigned long long)bases, mx, cudaGetErrorString(e));
}
// CK for buffers whose size long units drive
#define CKL(call, what) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) { if(!s.longs.empty()) return long_oom(s, e_, what); CK(e_); } } while(0)
// Device memory for hit lists sized past the default N ceiling's bound (a custom --n-ceil, or the re-run of a batch whose
// flags let more Ns through): CFB_ENOMEM naming the list length
static int hits_oom(const Slot& s, cudaError_t e) {
	cudaGetLastError();
	return fail(CFB_ENOMEM, "no device memory for the hit lists of a batch of %llu units whose mates may hold up to %u hits per strand "
	            "(reads up to %u bases under %s): %s", (unsigned long long)s.n_units, s.full_cap, s.maxlen,
	            s.custom_nceil ? "a custom --n-ceil" : "filter flags that let more Ns through", cudaGetErrorString(e));
}
#define CKH(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) { if(s.full_cap > s.maxlen / 4 + 8) return hits_oom(s, e_); CK(e_); } } while(0)

static int mate_too_long(uint64_t n, int m, const uint32_t* L) {
	for(uint64_t i = 0; i < n; i++)
		if(L[i] > kMaxMateLen) return fail(CFB_EINVAL, "unit %llu mate %d has %u bases: the limit is %u bases per mate", (unsigned long long)i, m + 1, L[i], kMaxMateLen);
	return CFB_OK;
}
// Units with a mate longer than kLongUnitLen go to the long-unit kernels (their flags are cleared for the others).  Returns the
// longest mate of the remaining units, which sizes the short kernels' buffers as before.
static uint32_t collect_longs(Slot& s, uint64_t n, int nm, const uint32_t* const len[2], const uint8_t* flags) {
	uint32_t mx = 0;
	for(uint64_t i = 0; i < n; i++) {
		const uint32_t l0 = len[0][i], l1 = nm == 2 ? len[1][i] : 0;
		if(l0 > kLongUnitLen || l1 > kLongUnitLen) s.longs.push_back(Slot::LongH{i, {l0, l1}, flags ? flags[i] : (uint8_t)3});
		else mx = std::max(mx, std::max(l0, l1));
	}
	return mx;
}

static int stage_batch(cfb_ctx* c, Slot& s, const cfb_batch* b) {
	if(!b || b->n_mates < 1 || b->n_mates > 2 || !b->bases || !b->off[0] || !b->len[0] || (b->n_mates == 2 && (!b->off[1] || !b->len[1])))
		return fail(CFB_EINVAL, "malformed cfb_batch");
	if(b->n_units >= (1ull << 30)) return fail(CFB_EINVAL, "batch too large (n_units must be < 2^30)");
	const uint64_t n = b->n_units; const int nm = b->n_mates;
	uint32_t maxlen = 0;
	for(int m = 0; m < nm; m++) {       // branch-free validation pass (vectorises); the offender is looked up only when there is one
		const uint64_t* O = b->off[m]; const uint32_t* L = b->len[m]; const uint64_t nb = b->n_bases; uint32_t mx = 0; uint64_t far = 0;
		for(uint64_t i = 0; i < n; i++) { const uint32_t l = L[i]; mx = l > mx ? l : mx; }
		if(mx > kMaxMateLen) return mate_too_long(n, m, L);
		for(uint64_t i = 0; i < n; i++) { const uint64_t e = O[i] + (uint64_t)L[i]; far = e > far ? e : far; }
		if(far > nb) { for(uint64_t i = 0; i < n; i++) if(O[i] + L[i] > nb) return fail(CFB_EINVAL, "unit %llu mate %d exceeds n_bases", (unsigned long long)i, m + 1); }
		maxlen = std::max(maxlen, mx);
	}
	s.longs.clear(); s.win_first = 0;
	if(maxlen > kLongUnitLen) maxlen = collect_longs(s, n, nm, b->len, b->flags);
	CKL(s.d_bases.ensure(b->n_bases + 16), "the bases"); CK(s.d_off.ensure(n * nm)); CK(s.d_len.ensure(n * nm)); CK(s.d_flags.ensure(n));
	// Caller arrays that already live in pinned memory (cfb_host_alloc) are DMA'd from where they are and
	// must stay untouched until cfb_classify_wait; pageable arrays are staged through pinned buffers first.
	const uint8_t* src_bases = b->bases;
	if(!is_pinned(b->bases)) { CK(s.h_bases.ensure(b->n_bases)); memcpy(s.h_bases.p, b->bases, b->n_bases); src_bases = s.h_bases.p; }
	CK(cudaMemcpyAsync(s.d_bases.p, src_bases, b->n_bases, cudaMemcpyHostToDevice, s.st));
	CK(s.h_off.ensure(n * nm)); CK(s.h_len.ensure(n * nm)); CK(s.h_flags.ensure(n));
	for(int m = 0; m < nm; m++) {
		const uint64_t* so = b->off[m]; const uint32_t* sl = b->len[m];
		if(!is_pinned(so)) { memcpy(s.h_off.p + m * n, so, n * 8); so = s.h_off.p + m * n; }
		if(!is_pinned(sl)) { memcpy(s.h_len.p + m * n, sl, n * 4); sl = s.h_len.p + m * n; }
		CK(cudaMemcpyAsync(s.d_off.p + m * n, so, n * 8, cudaMemcpyHostToDevice, s.st));
		CK(cudaMemcpyAsync(s.d_len.p + m * n, sl, n * 4, cudaMemcpyHostToDevice, s.st));
	}
	if(b->flags && is_pinned(b->flags)) CK(cudaMemcpyAsync(s.d_flags.p, b->flags, n, cudaMemcpyHostToDevice, s.st));
	else { if(b->flags) memcpy(s.h_flags.p, b->flags, n); else memset(s.h_flags.p, 3, n); CK(cudaMemcpyAsync(s.d_flags.p, s.h_flags.p, n, cudaMemcpyHostToDevice, s.st)); }
	s.bv.bases = s.d_bases.p; s.bv.flags = s.d_flags.p; s.bv.n_units = (uint32_t)n; s.bv.n_mates = nm;
	for(int m = 0; m < 2; m++) { s.bv.off[m] = m < nm ? s.d_off.p + m * n : nullptr; s.bv.len[m] = m < nm ? s.d_len.p + m * n : nullptr; }
	s.n_units = n; s.n_bases = b->n_bases; s.maxlen = maxlen;
	(void)c;
	return CFB_OK;
}

// ---------------------------------------------------------------------------------------
// Packed input (cfb_batch_packed): 2 bits per base + a sparse list of N positions instead of 1 byte per base, lengths
// instead of offsets -- about a third of the host->device bytes of cfb_batch.  The device expands it into the byte form
// the per-unit kernels read: every mate gets a 32-byte aligned slot of ceil(len/32)*32 bytes, so byte address =
// 32 * word index + base in word, for the unpack kernel and for the N list alike.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_wlen(const uint32_t* len, uint64_t n, uint32_t* wlen) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) wlen[i] = (len[i] + 31u) >> 5;
}
// thread per (mate slot, word k): 32 codes of one packed word -> 32 bytes
__global__ void __launch_bounds__(256) k_unpack(const uint64_t* __restrict__ words, const uint64_t* __restrict__ woff, uint64_t wbase, const uint32_t* __restrict__ len,
                                                uint64_t n, uint32_t W, uint8_t* bases, uint64_t* off) {
	const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(t >= n * W) return;
	const uint64_t i = t / W; const uint32_t k = (uint32_t)(t - i * W);
	const uint64_t w0 = wbase + woff[i];
	if(k == 0) off[i] = w0 * 32;
	if(k * 32 >= len[i]) return;
	const uint64_t w = __ldg(words + w0 + k);
	uint32_t o[8];
	#pragma unroll
	for(int q = 0; q < 8; q++) {          // 4 codes -> 4 bytes
		const uint32_t b = (uint32_t)(w >> (8 * q)) & 0xffu;
		o[q] = (b & 3u) | ((b & 0xcu) << 6) | ((b & 0x30u) << 12) | ((b & 0xc0u) << 18);
	}
	uint4* dst = reinterpret_cast<uint4*>(bases + (w0 + k) * 32);
	dst[0] = make_uint4(o[0], o[1], o[2], o[3]); dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
}
__global__ void __launch_bounds__(256) k_set_n(const uint64_t* npos, uint64_t n, uint8_t* bases, uint64_t limit) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < n) { const uint64_t p = npos[i]; if(p < limit) bases[p] = 4; }
}

static int stage_batch_packed(cfb_ctx* c, Slot& s, const cfb_batch_packed* b) {
	if(!b || b->n_mates < 1 || b->n_mates > 2 || !b->words || !b->len[0] || (b->n_mates == 2 && !b->len[1]) || (b->n_n && !b->n_pos))
		return fail(CFB_EINVAL, "malformed cfb_batch_packed");
	if(b->n_units >= (1ull << 30)) return fail(CFB_EINVAL, "batch too large (n_units must be < 2^30)");
	const uint64_t n = b->n_units; const int nm = b->n_mates;
	// one branch-free pass per mate over the lengths (it vectorises: this runs on the submitting thread, once per batch)
	uint32_t maxlen = 0; uint64_t need_words = 0, mate_words[2] = {0, 0};
	for(int m = 0; m < nm; m++) {
		const uint32_t* L = b->len[m]; uint32_t mx = 0; uint64_t w = 0;
		for(uint64_t i = 0; i < n; i++) { const uint32_t l = L[i]; mx = l > mx ? l : mx; w += (l + 31u) >> 5; }
		maxlen = std::max(maxlen, mx); mate_words[m] = w; need_words += w;
	}
	for(int m = 0; m < nm; m++) { const int rc = mate_too_long(n, m, b->len[m]); if(rc) return rc; }
	if(need_words != b->n_words) return fail(CFB_EINVAL, "cfb_batch_packed: n_words is %llu, the lengths need %llu", (unsigned long long)b->n_words, (unsigned long long)need_words);
	s.longs.clear(); s.win_first = 0;
	if(maxlen > kLongUnitLen) maxlen = collect_longs(s, n, nm, b->len, b->flags);
	const uint64_t scan_blocks = (n + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
	CKL(s.d_bases.ensure(b->n_words * 32 + 64), "the bases"); CK(s.d_off.ensure(n * nm + 1)); CK(s.d_len.ensure(n * nm)); CK(s.d_flags.ensure(n));
	CKL(s.d_words.ensure(b->n_words + 1), "the packed bases"); CK(s.d_npos.ensure(b->n_n + 1)); CK(s.d_wlen.ensure(n + 1)); CK(s.d_woff.ensure(n + 2)); CK(s.bsum.ensure(scan_blocks + 1));
	const uint64_t* src_words = b->words;
	if(!is_pinned(b->words)) { CK(s.h_words.ensure(b->n_words)); memcpy(s.h_words.p, b->words, b->n_words * 8); src_words = s.h_words.p; }
	CK(cudaMemcpyAsync(s.d_words.p, src_words, b->n_words * 8, cudaMemcpyHostToDevice, s.st));
	CK(s.h_len.ensure(n * nm)); CK(s.h_flags.ensure(n));
	for(int m = 0; m < nm; m++) {
		const uint32_t* sl = b->len[m];
		if(!is_pinned(sl)) { memcpy(s.h_len.p + m * n, sl, n * 4); sl = s.h_len.p + m * n; }
		CK(cudaMemcpyAsync(s.d_len.p + m * n, sl, n * 4, cudaMemcpyHostToDevice, s.st));
	}
	if(b->n_n) {
		const uint64_t* sp = b->n_pos;
		if(!is_pinned(sp)) { CK(s.h_off.ensure(b->n_n)); memcpy(s.h_off.p, sp, b->n_n * 8); sp = s.h_off.p; }
		CK(cudaMemcpyAsync(s.d_npos.p, sp, b->n_n * 8, cudaMemcpyHostToDevice, s.st));
	}
	if(b->flags && is_pinned(b->flags)) CK(cudaMemcpyAsync(s.d_flags.p, b->flags, n, cudaMemcpyHostToDevice, s.st));
	else { if(b->flags) memcpy(s.h_flags.p, b->flags, n); else memset(s.h_flags.p, 3, n); CK(cudaMemcpyAsync(s.d_flags.p, s.h_flags.p, n, cudaMemcpyHostToDevice, s.st)); }
	// expand on the device
	const uint32_t W = (maxlen + 31) / 32;
	uint64_t wbase = 0;
	CK(cudaMemsetAsync(s.scal.p + 5, 0, 8, s.st));
	for(int m = 0; m < nm && n; m++) {
		k_wlen<<<(unsigned)((n + 255) / 256), 256, 0, s.st>>>(s.d_len.p + m * n, n, s.d_wlen.p);
		k_scan_sums<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(s.d_wlen.p, n, s.bsum.p);
		k_scan_top<<<1, 1024, 0, s.st>>>(s.bsum.p, scan_blocks, (uint64_t*)(s.scal.p + 5));
		k_scan_apply<<<(unsigned)scan_blocks, kScanBlock, 0, s.st>>>(s.d_wlen.p, n, s.bsum.p, (const uint64_t*)(s.scal.p + 5), s.d_woff.p);
		if(W) k_unpack<<<(unsigned)((n * W + 255) / 256), 256, 0, s.st>>>(s.d_words.p, s.d_woff.p, wbase, s.d_len.p + m * n, n, W, s.d_bases.p, s.d_off.p + m * n);
		c->launches += 5;
		for(const Slot::LongH& l : s.longs) {      // W covers the other units: a long mate is expanded by a launch of its own
			const uint32_t Wl = (l.len[m] + 31) / 32;
			if(Wl <= W) continue;
			k_unpack<<<(unsigned)((Wl + 255) / 256), 256, 0, s.st>>>(s.d_words.p, s.d_woff.p + l.unit, wbase, s.d_len.p + m * n + l.unit, 1, Wl, s.d_bases.p, s.d_off.p + m * n + l.unit);
			c->launches++;
		}
		wbase += mate_words[m];      // mate 2 starts after all of mate 1
	}
	if(b->n_n) { k_set_n<<<(unsigned)((b->n_n + 255) / 256), 256, 0, s.st>>>(s.d_npos.p, b->n_n, s.d_bases.p, b->n_words * 32); c->launches++; }
	CK(cudaGetLastError());
	s.bv.bases = s.d_bases.p; s.bv.flags = s.d_flags.p; s.bv.n_units = (uint32_t)n; s.bv.n_mates = nm;
	for(int m = 0; m < 2; m++) { s.bv.off[m] = m < nm ? s.d_off.p + m * n : nullptr; s.bv.len[m] = m < nm ? s.d_len.p + m * n : nullptr; }
	s.n_units = n; s.n_bases = b->n_words * 32; s.maxlen = maxlen;
	return CFB_OK;
}

// The long units of the slot's window [win_first, win_first + n_units): their searched mates (tasks), with hit and segment
// space laid out by prefix sums over their own lengths, uploaded for the long-unit kernels.
static int long_plan(cfb_ctx* c, Slot& s) {
	s.nlong_win = 0; s.lntasks = 0; s.lhit_slots = 0; s.lsegs = 0; s.lmaxlen = 0;
	if(s.longs.empty()) return CFB_OK;
	const uint64_t lo = s.win_first, hi = s.win_first + s.n_units;
	CK(s.h_lunit.ensure(s.longs.size())); CK(s.h_ltask.ensure(2 * s.longs.size()));
	uint32_t nu = 0, nt = 0;
	for(const Slot::LongH& l : s.longs) {
		if(l.unit < lo || l.unit >= hi) continue;
		LongUnit u; u.unit = (uint32_t)(l.unit - lo); u.task0 = nt; u.ntask = 0; u.pad = 0;
		for(int m = 0; m < s.bv.n_mates; m++) {
			if(!((l.fl >> m) & 1) || l.len[m] == 0) continue;
			LongTask t; t.hoff = s.lhit_slots; t.soff = s.lsegs; t.unit = u.unit; t.mate = (uint32_t)m; t.len = l.len[m];
			t.nseg = (t.len + kSegLen - 1) / kSegLen;
			s.lhit_slots += 2ull * t.len; s.lsegs += 2ull * t.nseg; s.lmaxlen = std::max(s.lmaxlen, t.len);
			s.h_ltask.p[nt++] = t; u.ntask++;
		}
		s.h_lunit.p[nu++] = u;
	}
	s.nlong_win = nu; s.lntasks = nt;
	if(nu == 0) return CFB_OK;
	auto grow = [&](cudaError_t e) -> int {
		if(e == cudaSuccess) return CFB_OK;
		cudaGetLastError();
		return fail(CFB_ENOMEM, "no device memory for the long reads of this batch: %llu bases in %u long mates, the longest %u bases",
		            (unsigned long long)(s.lhit_slots / 2), nt, s.lmaxlen);
	};
	int rc;
	if((rc = grow(s.d_lunit.ensure(nu))) || (rc = grow(s.d_ltask.ensure(nt + 1))) || (rc = grow(s.lseg.ensure(s.lhit_slots + 1))) ||
	   (rc = grow(s.lhits.ensure(s.lhit_slots + 1))) || (rc = grow(s.lsn.ensure(s.lsegs + 1))) || (rc = grow(s.lsexit.ensure(s.lsegs + 1))) ||
	   (rc = grow(s.lnh.ensure(2ull * nt + 1))) || (rc = grow(s.lnrows.ensure(nu))) || (rc = grow(s.lroff.ensure(nu))) ||
	   (rc = grow(s.flags_short.ensure(s.n_units))) || (rc = grow(s.lstats.ensure(2)))) return rc;
	CK(cudaMemcpyAsync(s.d_lunit.p, s.h_lunit.p, nu * sizeof(LongUnit), cudaMemcpyHostToDevice, s.st));
	CK(cudaMemcpyAsync(s.d_ltask.p, s.h_ltask.p, nt * sizeof(LongTask), cudaMemcpyHostToDevice, s.st));
	CK(cudaMemsetAsync(s.lnh.p, 0, (2ull * nt + 1) * sizeof(uint32_t), s.st));
	CK(cudaMemsetAsync(s.lstats.p, 0, 2 * sizeof(unsigned long long), s.st));
	CK(cudaMemcpyAsync(s.flags_short.p, s.bv.flags, s.n_units, cudaMemcpyDeviceToDevice, s.st));
	k_mask_long<<<(nu + 127) / 128, 128, 0, s.st>>>(s.d_lunit.p, nu, s.flags_short.p); c->launches++;
	return CFB_OK;
}

// Enqueue all kernels of one batch on the slot's stream.  stage: 0 = from search, 1 = from k_rows
// (after a rows-capacity overflow; the hit lists are already post-processed and sorted).
static int enqueue_kernels(cfb_ctx* c, Slot& s, int stage, bool time_it) {
	const uint64_t n = s.n_units; const int nm = s.bv.n_mates;
	const uint64_t ntasks = n * nm * 2;
	if(stage == 0 && n) { const int rc = long_plan(c, s); if(rc) return rc; }
	BatchView sb = s.bv;                 // what the short kernels see: the long units' flags cleared
	if(s.nlong_win) sb.flags = s.flags_short.p;
	const uint32_t ublocks = (uint32_t)((n + 127) / 128);
	const uint64_t scan_blocks = (n + kScanBlock * kScanPer - 1) / (kScanBlock * kScanPer);
	if(n == 0) return CFB_OK;
	// which search kernel runs decides what it stores: k_search_t keeps only hits of >= kLongLen bases when min_hitlen allows
	// it (see kListRegen); k_search_long -- for long reads, and the scalar search of a CFB_COUNT=1 pass at any read length --
	// and small min_hitlen keep every hit
	const SearchKernel search = search_kernel(s.maxlen, c->count, c->view.cr != nullptr);
	const bool keep_short = search == k_search_long<true> || search == k_search_long<false> || search == k_search_long<false, true> || c->prm.min_hitlen < kLongLen || c->keep_short;
	if(stage == 0) {
		if(s.cap == 0) {
			s.full_cap = s.maxlen / 4 + 8;      // >= #Ns allowed by the N filter (0.15 len) + len/10 + slack
			if(s.custom_nceil) s.full_cap = nceil_full_cap(s.nceil, s.maxlen);
			s.cap = keep_short ? s.full_cap : s.maxlen / kLongLen + 2;       // hits of >= 22 bases do not overlap
		}
		CKH(s.hits.ensure(ntasks * s.cap)); CK(s.nhits.ensure(ntasks));
		if(!keep_short) {
			s.regen_slots = std::max<uint64_t>(s.regen_slots, c->regen_slots0 ? c->regen_slots0 : std::max<uint64_t>(ntasks / 32, 1024));
			CKH(s.regen.ensure(s.regen_slots * s.full_cap)); CK(s.regen_n.ensure(s.regen_slots));
			CK(cudaMemsetAsync(s.scal.p + 6, 0, sizeof(unsigned long long), s.st));
		}
		const uint32_t W = (s.maxlen + 31) / 32 + 1;
		CK(s.pk.ensure(ntasks * W + 2)); CK(s.nm.ensure(ntasks * W + 2)); CK(s.nrows.ensure(n)); CK(s.row_off.ensure(n + 1));
		CK(s.bsum.ensure(scan_blocks + 1)); CK(s.nout.ensure(n + 1)); CK(s.out_off.ensure(n + 1)); CK(s.rec_off32.ensure(n + 1));
		s.rows_cap = std::max<uint64_t>(s.rows_cap, c->rows_cap0 ? c->rows_cap0 : std::max<uint64_t>(n * 12, 4096));
	}
	if(s.nlong_win) {
		CKL(s.rows.ensure(s.rows_cap), "the rows"); CKL(s.ids.ensure(s.rows_cap), "the rows"); CKL(s.entries.ensure(s.rows_cap), "the hit maps");
		CKL(s.tcs.ensure(s.rows_cap), "the hit maps"); CKL(s.sparse.ensure(s.rows_cap), "the records"); CKL(s.dense.ensure(s.rows_cap), "the records");
		CKL(s.lhl.ensure(s.rows_cap), "the rows");
	}
	CK(s.rows.ensure(s.rows_cap)); CK(s.ids.ensure(s.rows_cap)); CK(s.entries.ensure(s.rows_cap)); CK(s.tcs.ensure(s.rows_cap)); CK(s.sparse.ensure(s.rows_cap));
	s.dense_cap = s.rows_cap; CK(s.dense.ensure(s.dense_cap));
	CK(cudaMemsetAsync(s.scal.p, 0, 4 * sizeof(unsigned long long), s.st));   // task counters, overflow flag, row allocator; [4] is rewritten by the scan
	if(time_it) CK(cudaEventRecord(s.ev[0], s.st));
	Counters* ctr = c->count ? c->d_ctr.p : nullptr;
	if(c->count && stage == 0) CK(cudaMemsetAsync(c->d_ctr.p, 0, sizeof(Counters), s.st));
	else if(c->count) {      // a re-run from the row stage scores every unit again: its k_score statistics start over
		const size_t sc0 = offsetof(Counters, sc_units);
		CK(cudaMemsetAsync(reinterpret_cast<char*>(c->d_ctr.p) + sc0, 0, sizeof(Counters) - sc0, s.st));
	}
	UnitArgs ua; ua.v = c->view; ua.p = c->prm; ua.b = sb; ua.hits = s.hits.p; ua.nhits = s.nhits.p; ua.cap = s.cap;
	ua.nrows = s.nrows.p; ua.row_off = s.row_off.p; ua.row_total = s.scal.p + 3; ua.rows = s.rows.p; ua.ids = s.ids.p; ua.rows_cap = s.rows_cap;
	ua.entries = s.entries.p; ua.tcs = s.tcs.p; ua.recs_sparse = s.sparse.p; ua.nout = s.nout.p;
	ua.overflow = (unsigned int*)(s.scal.p + 2); ua.ctr = ctr;
	ua.regen = s.regen.p; ua.regen_n = s.regen_n.p; ua.regen_ctr = s.scal.p + 6; ua.regen_slots = s.regen_slots; ua.full_cap = s.full_cap; ua.keep_short = keep_short ? 1u : 0u;
	if(stage == 0) {
		SearchArgs sa; sa.v = c->view; sa.p = c->prm; sa.b = sb; sa.hits = s.hits.p; sa.nhits = s.nhits.p; sa.cap = s.cap;
		const uint32_t W = (s.maxlen + 31) / 32 + 1;
		sa.pk = s.pk.p; sa.nm = s.nm.p; sa.W = W; sa.keep_short = keep_short ? 1u : 0u;
		{ PackArgs pa; pa.b = sb; pa.pk = s.pk.p; pa.nm = s.nm.p; pa.W = W;
		  k_pack<<<(unsigned)((ntasks * W + 127) / 128), 128, 0, s.st>>>(pa); c->launches++; }
		sa.task_ctr64 = s.scal.p + 0; sa.ntasks = (uint32_t)ntasks; sa.overflow = (unsigned int*)(s.scal.p + 2); sa.ctr = ctr;
		int occ = 1;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, search, kSearchThreads, 0));
		const uint64_t resident = (uint64_t)c->ix->sm_count * (uint64_t)std::max(occ, 1);
		const uint64_t warps = resident * (kSearchThreads / 32);
		sa.chunk = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(ntasks / (warps * 4), 32), 256);      // k_search_t: one atomic per warp refill of >= 32 tasks
		const int blocks = (int)std::min<uint64_t>(resident, (ntasks + kSearchThreads - 1) / kSearchThreads);
		search<<<blocks, kSearchThreads, 0, s.st>>>(sa);
		c->launches++;
		if(time_it) CK(cudaEventRecord(s.ev[1], s.st));
		k_prep<8, false><<<ublocks, 128, 0, s.st>>>(ua); c->launches++;          // <= 64 registers (measured best of 72 / 64 / 40)
	} else {
		if(time_it) CK(cudaEventRecord(s.ev[1], s.st));
		k_prep<8, true><<<ublocks, 128, 0, s.st>>>(ua); c->launches++;
	}
	LongArgs la;
	if(s.nlong_win) {
		la.v = c->view; la.p = c->prm; la.b = s.bv; la.tasks = s.d_ltask.p; la.ntasks = s.lntasks; la.units = s.d_lunit.p; la.nunits = s.nlong_win;
		la.nsegs = s.lsegs; la.seg = s.lseg.p; la.sn = s.lsn.p; la.sexit = s.lsexit.p; la.hits = s.lhits.p; la.nh = s.lnh.p;
		la.nrows = s.lnrows.p; la.roff = s.lroff.p; la.hl = s.lhl.p; la.stats = s.lstats.p; la.u = ua;
		const unsigned ub = (s.nlong_win + 31) / 32;
		if(stage == 0) {
			if(s.lntasks) {
				if(c->count == 1) k_long_join<true><<<(2 * s.lntasks + 127) / 128, 128, 0, s.st>>>(la);
				else {
					k_long_seg<<<(unsigned)((s.lsegs + 127) / 128), 128, 0, s.st>>>(la);
					k_long_join<false><<<(2 * s.lntasks + 127) / 128, 128, 0, s.st>>>(la);
				}
				k_long_post<<<(s.lntasks + 127) / 128, 128, 0, s.st>>>(la);
				c->launches += c->count == 1 ? 2 : 3;
			}
			k_long_prep<false><<<ub, 32, 0, s.st>>>(la);
		} else k_long_prep<true><<<ub, 32, 0, s.st>>>(la);
		c->launches++;
	}
	if(time_it) CK(cudaEventRecord(s.ev[2], s.st));
	ResolveArgs ra; ra.v = c->view; ra.rows = s.rows.p; ra.ids = s.ids.p; ra.ids16 = nullptr; ra.total = (const uint64_t*)(s.scal.p + 3); ra.rows_cap = s.rows_cap;
	ra.task_ctr = s.scal.p + 1; ra.chunk = 64; ra.ctr = ctr;
	if((c->view.rtab16 || c->view.rtab32) && c->count != 1) k_lookup<<<c->ix->sm_count * 8, 256, 0, s.st>>>(ra);
	else if(c->view.cr) { if(c->count) k_resolve_c<true, false, true><<<c->resolve_blocks, kSearchThreads, 0, s.st>>>(ra); else k_resolve_c<false, false, true><<<c->resolve_blocks, kSearchThreads, 0, s.st>>>(ra); }
	else if(c->count) k_resolve_c<true, false><<<c->resolve_blocks, kSearchThreads, 0, s.st>>>(ra);
	else k_resolve_c<false, false><<<c->resolve_blocks, kSearchThreads, 0, s.st>>>(ra);
	c->launches++;
	if(time_it) CK(cudaEventRecord(s.ev[3], s.st));
	if(ctr) k_score<12, true><<<ublocks, kScoreThreads, 0, s.st>>>(ua);
	else k_score<12, false><<<ublocks, kScoreThreads, 0, s.st>>>(ua);        // <= 40 registers and 14.5 KB of shared memory: 12 CTAs per SM
	if(s.nlong_win) { k_long_score<<<(s.nlong_win + 127) / 128, 128, 0, s.st>>>(la); c->launches++; }
	// record offsets: one single-pass scan over the n + 1 counts (the last is 0, so out_off[n] is the total), in 64 bits
	size_t scan_bytes = 0;
	CK(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, s.nout.p, s.out_off.p, cub::Sum(), (uint64_t)0, (int)(n + 1), s.st));
	CK(s.scan_tmp.ensure(scan_bytes));
	CK(cudaMemsetAsync(s.nout.p + n, 0, sizeof(uint32_t), s.st));
	CK(cub::DeviceScan::ExclusiveScan(s.scan_tmp.p, scan_bytes, s.nout.p, s.out_off.p, cub::Sum(), (uint64_t)0, (int)(n + 1), s.st));
	CK(cudaMemcpyAsync(s.scal.p + 4, s.out_off.p + n, sizeof(uint64_t), cudaMemcpyDeviceToDevice, s.st));
	k_compact<<<(unsigned)((n + 1 + 127) / 128), 128, 0, s.st>>>((uint32_t)n, s.row_off.p, s.out_off.p, s.sparse.p, s.dense.p, s.rec_off32.p, s.dense_cap, (unsigned int*)(s.scal.p + 2));
	c->launches += 4;      // k_score, the scan's two kernels, k_compact
	s.folded = false;
	if(c->fold_records && !s.is_text) {      // this batch's per-taxon counters, on the device, from the records just written
		const uint32_t nsp = c->cnt.n;
		CK(s.cnt.ensure(3ull * nsp)); CK(cudaMemsetAsync(s.cnt.p, 0, 3ull * nsp * 8, s.st));
		FoldArgs fa; fa.sp_taxid = c->cnt.d_taxid.p; fa.n_sp = nsp; fa.rec_off = s.rec_off32.p; fa.recs = s.dense.p; fa.n_units = (uint32_t)n; fa.n_mates = nm;
		fa.khits = c->prm.khits; fa.len[0] = s.bv.len[0]; fa.len[1] = s.bv.len[1]; fa.flags = s.bv.flags; fa.sp = s.cnt.p;
		k_fold_counts<<<ublocks, 128, 0, s.st>>>(fa); c->launches++;
		s.folded = true;
	}
	if(time_it) CK(cudaEventRecord(s.ev[4], s.st));
	s.d2h_recs = 0;
	if(s.want_host) {
		// results go home behind the kernels without waiting for the host to learn their size: record offsets
		// exactly, records for the count the previous batches suggest (finish_batch fetches a remainder if any)
		const uint64_t guess = std::min<uint64_t>(s.dense_cap, (uint64_t)((double)n * c->rec_ratio * 1.05) + 4096);
		CK(s.h_recs.ensure(guess + 1)); CK(s.h_rec_off.ensure(n + 1));
		CK(cudaMemcpyAsync(s.h_rec_off.p, s.rec_off32.p, (n + 1) * 4, cudaMemcpyDeviceToHost, s.st));
		CK(cudaMemcpyAsync(s.h_recs.p, s.dense.p, guess * sizeof(OutRec), cudaMemcpyDeviceToHost, s.st));
		s.d2h_recs = guess;
	}
	CK(cudaMemcpyAsync(s.h_scal.p, s.scal.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s.st));
	CK(cudaGetLastError());
	return CFB_OK;
}

// Wait for the kernels, handle capacity overflows by re-running the affected stages, then D2H.
static int finish_batch(cfb_ctx* c, Slot& s, bool time_it, bool to_host, cfb_result* out) {
	if(s.n_units == 0) { if(out) { out->n_units = 0; out->n_recs = 0; out->rec_off = nullptr; out->recs = nullptr; } return CFB_OK; }
	for(int attempt = 0; attempt < 8; attempt++) {
		CK(cudaStreamSynchronize(s.st));
		const unsigned ovf = (unsigned)(s.h_scal.p[2] & 0xffffffffu);
		const uint64_t total_rows = s.h_scal.p[3];
		if(ovf == 4) {            // more lists needed regeneration than the side buffer holds: h_scal[6] tells how many
			s.regen_slots = s.h_scal.p[6] + s.h_scal.p[6] / 4 + 1024; s.reran = true;
			int rc = enqueue_kernels(c, s, 0, time_it); if(rc) return rc;
			continue;
		}
		if(ovf == 1) {            // hit-list capacity: the caller's flags let more Ns through than the context's ceiling bounds
			s.cap = s.maxlen + 2; s.full_cap = s.maxlen + 2; s.reran = true;
			int rc = enqueue_kernels(c, s, 0, time_it); if(rc) return rc;
			continue;
		}
		if(total_rows > s.rows_cap) {
			s.rows_cap = total_rows + total_rows / 4 + 1024; s.reran = true;
			int rc = enqueue_kernels(c, s, 1, time_it); if(rc) return rc;
			continue;
		}
		if(ovf != 0) return fail(CFB_ECUDA, "internal capacity error %u", ovf);
		break;
	}
	const uint64_t nrec = s.h_scal.p[4];
	c->regen_lists += s.h_scal.p[6]; c->regen_tasks += (uint64_t)s.n_units * (uint64_t)s.bv.n_mates * 2;
	if(s.nlong_win) {
		unsigned long long st[2];
		CK(cudaMemcpy(st, s.lstats.p, sizeof st, cudaMemcpyDeviceToHost));
		c->long_units += s.nlong_win; c->long_bases += s.lhit_slots / 2; c->long_searches += st[0]; c->long_researched += st[1];
	}
	if(s.folded) {        // the batch is final: add its counters to the context's totals (stream order keeps this ahead of any read)
		const uint32_t n3 = 3 * c->cnt.n;
		k_cnt_commit<<<(n3 + 255) / 256, 256, 0, s.st>>>(s.cnt.p, c->cnt.total.p, n3); c->launches++;
		CK(cudaEventRecord(s.ev[5], s.st)); s.commit_pending = true;       // cfb_counts_allreduce orders itself behind this event, without a host-side wait
		s.folded = false; c->cnt.reduced = false;
	}
	if(to_host) {
		if(s.n_units) c->rec_ratio = std::max(c->rec_ratio * 0.98, (double)nrec / (double)s.n_units);
		if(!s.want_host || nrec > s.d2h_recs) {       // not (fully) covered by the speculative copy
			const uint64_t have = s.want_host ? s.d2h_recs : 0;
			if(nrec + 1 > s.h_recs.cap) {             // grow, keeping nothing: copy everything again
				CK(s.h_recs.ensure(nrec + 1));
				if(nrec) CK(cudaMemcpyAsync(s.h_recs.p, s.dense.p, nrec * sizeof(OutRec), cudaMemcpyDeviceToHost, s.st));
			} else if(nrec > have) CK(cudaMemcpyAsync(s.h_recs.p + have, s.dense.p + have, (nrec - have) * sizeof(OutRec), cudaMemcpyDeviceToHost, s.st));
			if(!s.want_host) { CK(s.h_rec_off.ensure(s.n_units + 1)); CK(cudaMemcpyAsync(s.h_rec_off.p, s.rec_off32.p, (s.n_units + 1) * 4, cudaMemcpyDeviceToHost, s.st)); }
			CK(cudaStreamSynchronize(s.st));
		}
	}
	if(out) { out->n_units = s.n_units; out->n_recs = nrec; out->rec_off = s.h_rec_off.p; out->recs = reinterpret_cast<const cfb_rec*>(s.h_recs.p); }
	return CFB_OK;
}

extern "C" int cfb_classify_submit(cfb_ctx* c, int slot, const cfb_batch* b) {
	if(!c || slot < 0 || slot >= kSlots - 1) return fail(CFB_EINVAL, "bad ctx/slot");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[slot];
	if(s.pending) return fail(CFB_EINVAL, "slot %d still has an un-waited batch", slot);
	int rc = stage_batch(c, s, b); if(rc) return rc;
	s.cap = 0; s.want_host = true; s.is_text = false; s.nceil = c->nceil; s.custom_nceil = !c->nceil.is_default();
	rc = enqueue_kernels(c, s, 0, false); if(rc) return rc;
	s.pending = true;
	return CFB_OK;
}
extern "C" int cfb_classify_submit_packed(cfb_ctx* c, int slot, const cfb_batch_packed* b) {
	if(!c || slot < 0 || slot >= kSlots - 1) return fail(CFB_EINVAL, "bad ctx/slot");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[slot];
	if(s.pending) return fail(CFB_EINVAL, "slot %d still has an un-waited batch", slot);
	int rc = stage_batch_packed(c, s, b); if(rc) return rc;
	s.cap = 0; s.want_host = true; s.is_text = false; s.nceil = c->nceil; s.custom_nceil = !c->nceil.is_default();
	rc = enqueue_kernels(c, s, 0, false); if(rc) return rc;
	s.pending = true;
	return CFB_OK;
}
// Host helper: the packed form of a cfb_batch (single pass, one thread; callers that parse reads themselves can emit
// the packed form directly).  Returns CFB_EINVAL when a capacity is too small; n_words / n_n always receive the sizes needed.
extern "C" int cfb_pack_batch(const cfb_batch* in, uint64_t* words, uint64_t words_cap, uint64_t* n_pos, uint64_t npos_cap, uint64_t* n_words, uint64_t* n_n) {
	if(!in || !n_words || !n_n || in->n_mates < 1 || in->n_mates > 2) return fail(CFB_EINVAL, "cfb_pack_batch: bad argument");
	uint64_t w = 0, nn = 0; bool fits = true;
	for(int m = 0; m < in->n_mates; m++) for(uint64_t i = 0; i < in->n_units; i++) {
		const uint8_t* p = in->bases + in->off[m][i]; const uint32_t len = in->len[m][i];
		for(uint32_t k = 0; k < len; k += 32) {
			uint64_t v = 0; const uint32_t cnt = std::min<uint32_t>(32, len - k);
			for(uint32_t j = 0; j < cnt; j++) {
				const uint8_t c = p[k + j];
				if(c > 3) { if(n_pos && nn < npos_cap) n_pos[nn] = (w << 5) | j; else fits = false; nn++; }
				else v |= (uint64_t)c << (2 * j);
			}
			if(words && w < words_cap) words[w] = v; else fits = false;
			w++;
		}
	}
	*n_words = w; *n_n = nn;
	return fits ? CFB_OK : fail(CFB_EINVAL, "cfb_pack_batch: buffers too small (%llu words, %llu N positions needed)", (unsigned long long)w, (unsigned long long)nn);
}
extern "C" int cfb_classify_wait(cfb_ctx* c, int slot, cfb_result* out) {
	if(!c || slot < 0 || slot >= kSlots - 1 || !out) return fail(CFB_EINVAL, "bad ctx/slot");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[slot];
	if(!s.pending) return fail(CFB_EINVAL, "slot %d has no submitted batch", slot);
	s.pending = false;
	return finish_batch(c, s, false, true, out);
}
extern "C" int cfb_classify_batch(cfb_ctx* c, const cfb_batch* b, cfb_result* out) {
	int rc = cfb_classify_submit(c, 0, b); if(rc) return rc;
	return cfb_classify_wait(c, 0, out);
}

extern "C" int cfb_batch_upload(cfb_ctx* c, const cfb_batch* b, cfb_dbatch** out) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	if(c->resident_used) return fail(CFB_EINVAL, "only one resident batch per ctx");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[kSlots - 1];
	int rc = stage_batch(c, s, b); if(rc) return rc;
	CK(cudaStreamSynchronize(s.st));
	s.cap = 0; s.is_text = false; s.nceil = c->nceil; s.custom_nceil = !c->nceil.is_default();
	c->resident.slot = kSlots - 1; c->resident.n_units = s.n_units; c->resident_used = true;
	*out = &c->resident;
	return CFB_OK;
}
extern "C" void cfb_dbatch_free(cfb_ctx* c, cfb_dbatch*) { if(c) c->resident_used = false; }
extern "C" int cfb_classify_resident(cfb_ctx* c, cfb_dbatch* d, float* ms, uint64_t* n_recs) {
	return cfb_classify_resident_range(c, d, 0, d ? d->n_units : 0, ms, n_recs);
}
extern "C" int cfb_classify_resident_range(cfb_ctx* c, cfb_dbatch* d, uint64_t first, uint64_t count, float* ms, uint64_t* n_recs) {
	if(!c || !d) return fail(CFB_EINVAL, "null argument");
	if(first + count > d->n_units) return fail(CFB_EINVAL, "cfb_classify_resident_range: units [%llu, %llu) exceed the uploaded batch", (unsigned long long)first, (unsigned long long)(first + count));
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[d->slot];
	// a window of the uploaded batch: offsets are absolute into the uploaded bases, so only the per-unit arrays shift
	const uint64_t N = d->n_units; const int nmates = s.bv.n_mates;
	s.bv.flags = s.d_flags.p + first; s.bv.n_units = (uint32_t)count; s.n_units = count; s.win_first = first;
	for(int m = 0; m < nmates; m++) { s.bv.off[m] = s.d_off.p + m * N + first; s.bv.len[m] = s.d_len.p + m * N + first; }
	int rc = enqueue_kernels(c, s, 0, true); if(rc) return rc;
	cfb_result r;
	rc = finish_batch(c, s, true, false, &r); if(rc) return rc;
	if(n_recs) *n_recs = r.n_recs;
	if(ms) {
		CK(cudaEventSynchronize(s.ev[4]));
		CK(cudaEventElapsedTime(&ms[0], s.ev[0], s.ev[1])); CK(cudaEventElapsedTime(&ms[1], s.ev[1], s.ev[2]));
		CK(cudaEventElapsedTime(&ms[2], s.ev[2], s.ev[3])); CK(cudaEventElapsedTime(&ms[3], s.ev[3], s.ev[4]));
		CK(cudaEventElapsedTime(&ms[4], s.ev[0], s.ev[4]));
	}
	return CFB_OK;
}
extern "C" int cfb_resident_result(cfb_ctx* c, cfb_result* out) {
	if(!c || !out || !c->resident_used) return fail(CFB_EINVAL, "no resident batch");
	CK(cudaSetDevice(c->ix->device));
	Slot& s = c->slots[kSlots - 1];
	return finish_batch(c, s, false, true, out);
}
extern "C" int cfb_ctx_long_stats(const cfb_ctx* c, uint64_t out[4]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	out[0] = c->long_units; out[1] = c->long_bases; out[2] = c->long_searches; out[3] = c->long_researched;
	return CFB_OK;
}
extern "C" int cfb_ctx_counters(cfb_ctx* c, uint64_t out[8]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	Counters h; CK(cudaMemcpy(&h, c->d_ctr.p, sizeof h, cudaMemcpyDeviceToHost));
	out[0] = h.units; out[1] = h.partial_searches; out[2] = h.ftab_probes; out[3] = h.sides_search;
	out[4] = h.walk_steps; out[5] = h.rows_resolved; out[6] = h.lf_steps; out[7] = h.ext_searches;
	return CFB_OK;
}

// pinned for every device of the process (several contexts on different GPUs may DMA from the same buffer pool)
extern "C" void* cfb_host_alloc(size_t bytes) { void* p = nullptr; if(cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
extern "C" int cfb_device_count(void) { int n = 0; if(cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }
extern "C" void cfb_host_free(void* p) { if(p) cudaFreeHost(p); }

extern "C" int cfb_test_lf(const cfb_index* ix, const uint64_t* rows, const uint8_t* chars, uint64_t n, uint64_t* out) {
	if(!ix || ix->device < 0) return fail(CFB_ENODEV, "no device");
	CK(cudaSetDevice(ix->device));
	DBuf<uint64_t> dr, dout; DBuf<uint8_t> dc;
	CK(dr.alloc(n + 1)); CK(dout.alloc(n + 1)); CK(dc.alloc(n + 8));
	CK(cudaMemcpy(dr.p, rows, n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dc.p, chars, n, cudaMemcpyHostToDevice));
	k_test_lf<<<64, 128>>>(ix->view, dr.p, dc.p, n, dout.p);
	CK(cudaDeviceSynchronize());
	CK(cudaMemcpy(out, dout.p, n * 8, cudaMemcpyDeviceToHost));
	return CFB_OK;
}
extern "C" int cfb_test_resolve(const cfb_index* ix, const uint64_t* rows, uint64_t n, uint32_t* out) {
	if(!ix || ix->device < 0) return fail(CFB_ENODEV, "no device");
	CK(cudaSetDevice(ix->device));
	DBuf<uint64_t> dr; DBuf<uint32_t> dout; DBuf<unsigned long long> sc;
	CK(dr.alloc(n + 1)); CK(dout.alloc(n + 2)); CK(sc.alloc(2));
	CK(cudaMemcpy(dr.p, rows, n * 8, cudaMemcpyHostToDevice));
	unsigned long long init[2] = {0ull, (unsigned long long)n};
	CK(cudaMemcpy(sc.p, init, 16, cudaMemcpyHostToDevice));
	ResolveArgs ra; ra.v = ix->view; ra.rows = dr.p; ra.ids = dout.p; ra.ids16 = nullptr; ra.total = (const uint64_t*)(sc.p + 1); ra.rows_cap = n; ra.task_ctr = sc.p; ra.chunk = 64; ra.ctr = nullptr;
	if(ix->view.cr) k_resolve_c<false, false, true><<<32, kSearchThreads>>>(ra);
	else k_resolve_c<false, false><<<32, kSearchThreads>>>(ra);
	CK(cudaDeviceSynchronize());
	CK(cudaMemcpy(out, dout.p, n * 4, cudaMemcpyDeviceToHost));
	return CFB_OK;
}

#include "cf_text.cuh"
#include "cf_multi.cuh"

cfb_ctx::~cfb_ctx() {
	if(ix && ix->device >= 0) cudaSetDevice(ix->device);
	for(int i = 0; i < kSlots; i++) if(slots[i].st) cudaStreamSynchronize(slots[i].st);
	if(comm_st) cudaStreamSynchronize(comm_st);
	if(getenv("CFB_REGEN_STATS") && regen_tasks)
		fprintf(stderr, "[cfb] strand lists regenerated by k_prep: %llu of %llu (%.3f %%)\n", (unsigned long long)regen_lists,
		        (unsigned long long)regen_tasks, 100.0 * (double)regen_lists / (double)regen_tasks);
	if(comm && g_nccl.lib) g_nccl.CommDestroy((ncclComm_t)comm);
}

// Test hook: the device's double log and sqrt of every integer length in [lo, hi) against the host's (glibc), bit for
// bit -- what cf_nceil.h's G and S ceilings rely on.  Counts the mismatches, and in n_log_far the logs more than one unit
// in the last place apart; first_log: the first length whose log differs.
__global__ void k_test_log_sqrt(uint64_t lo, uint64_t n, unsigned long long* lg, unsigned long long* sq) {
	const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
	if(i >= n) return;
	const double x = (double)(lo + i);
	lg[i] = (unsigned long long)__double_as_longlong(log(x)); sq[i] = (unsigned long long)__double_as_longlong(__dsqrt_rn(x));
}
extern "C" int cfb_test_log_sqrt(int device, uint64_t lo, uint64_t hi, uint64_t* n_log, uint64_t* n_log_far, uint64_t* n_sqrt, uint64_t* first_log) {
	if(!n_log || !n_log_far || !n_sqrt || !first_log || hi < lo) return fail(CFB_EINVAL, "cfb_test_log_sqrt: bad argument");
	CK(cudaSetDevice(device));
	const uint64_t chunk = 1ull << 26;
	DBuf<unsigned long long> dl, ds; HBuf<unsigned long long> hl, hs;
	CK(dl.ensure(chunk)); CK(ds.ensure(chunk)); CK(hl.ensure(chunk)); CK(hs.ensure(chunk));
	std::atomic<uint64_t> bad_l(0), bad_s(0), far_l(0); uint64_t first = UINT64_MAX;
	const int nth = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
	for(uint64_t a = lo; a < hi; a += chunk) {
		const uint64_t n = std::min(chunk, hi - a);
		k_test_log_sqrt<<<(unsigned)((n + 255) / 256), 256>>>(a, n, dl.p, ds.p);
		CK(cudaMemcpy(hl.p, dl.p, n * 8, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(hs.p, ds.p, n * 8, cudaMemcpyDeviceToHost));
		std::vector<uint64_t> firsts(nth, UINT64_MAX); std::vector<std::thread> th;
		for(int t = 0; t < nth; t++) th.emplace_back([&, t]() {
			uint64_t bl = 0, bs = 0, fl = 0;
			for(uint64_t i = t; i < n; i += nth) {
				const double x = (double)(a + i), l = std::log(x), s = std::sqrt(x);
				unsigned long long ul, us; memcpy(&ul, &l, 8); memcpy(&us, &s, 8);
				if(ul != hl.p[i]) { bl++; firsts[t] = std::min<uint64_t>(firsts[t], a + i); if(ul + 1 != hl.p[i] && ul != hl.p[i] + 1) fl++; }
				if(us != hs.p[i]) bs++;
			}
			bad_l += bl; bad_s += bs; far_l += fl;
		});
		for(std::thread& x : th) x.join();
		for(uint64_t f : firsts) first = std::min(first, f);
	}
	*n_log = bad_l; *n_log_far = far_l; *n_sqrt = bad_s; *first_log = first;
	return CFB_OK;
}
