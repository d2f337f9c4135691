// cf_kernels.cuh -- shared declarations of the sm_90a kernels of the classification path (cfb200.cu).
//
// Work decomposition (one batch of units = reads or pairs), DESIGN.md section 4:
//   k_pack       reads (1 byte/base) -> 2-bit strands in search order + N masks
//   k_search_t   FM-index backward search, the hot loop: ONE THREAD per (unit, mate, strand) greedy walk over the
//                re-cut device index (rank16: one 16-byte gather per rank query; K-mer (with its death bitmap) and walk8 tables
//                delete dependent gathers); one fetch point per loop iteration for all 32 walks of a warp
//   k_search<G>  the warp-cooperative A/B variant (G lanes per walk on the file's 128-byte sides, shuffle popcount):
//                same results, issue-bound and several times slower; uses the
//                cooperative side primitives below
//   k_prep       thread per unit: extend / twin-removal / trim, strand choice, libstdc++-exact sort, row allocation,
//                rows with the scoring plan in their high bits
//   k_lookup / k_resolve_c   SA row -> sequence id (table gather / 4-lane walk-left on rank16)
//   k_score      thread per unit: hit map, score finalisation, host rule, taxonomy-tree reduction, emit
//   k_scan_*, k_compact, k_fold_counts   offsets, dense records, per-taxon counters
#ifndef CF_KERNELS_CUH_
#define CF_KERNELS_CUH_

#include <cuda_runtime.h>
#include "cf_logic.h"

namespace cfb {

struct BatchView {
	const uint8_t*  bases;
	const uint64_t* off[2];
	const uint32_t* len[2];
	const uint8_t*  flags;     // may be null
	uint32_t n_units; int32_t n_mates;
};

static const int kGroup = 8;           // lanes per walk
static const int kSearchThreads = 128; // 4 warps = 16 walks per CTA

// --------------------------------------------------------------------------------------
// cooperative side primitives (8 lanes, lane gl holds bytes [16*gl, 16*gl+16) of the side)
// --------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t sel_word(const uint4& d, uint32_t k) {
	return k == 0 ? d.x : (k == 1 ? d.y : (k == 2 ? d.z : d.w));
}
// matches of 2-bit code c among the first n (0..64) bases of this lane's 16 bytes
__device__ __forceinline__ uint32_t lane_count(const uint4& d, uint32_t rep, int n) {
	uint32_t r = 0;
	#pragma unroll
	for(int k = 0; k < 4; k++) {
		const uint32_t w = sel_word(d, k);
		const uint32_t y = ~(w ^ rep);
		const uint32_t m = y & (y >> 1) & 0x55555555u;
		int nk = n - 16 * k; nk = nk < 0 ? 0 : (nk > 16 ? 16 : nk);
		const uint32_t mask = nk == 0 ? 0u : (0xFFFFFFFFu >> (32 - 2 * nk));
		r += __popc(m & mask);
	}
	return r;
}
__device__ __forceinline__ uint32_t group_sum(uint32_t x, unsigned gmask) {
	x += __shfl_xor_sync(gmask, x, 1);
	x += __shfl_xor_sync(gmask, x, 2);
	x += __shfl_xor_sync(gmask, x, 4);
	return x;
}
// occ[c] of the side whose 16-byte pieces are in d: lanes 6,7 hold {A,C},{G,T}
__device__ __forceinline__ uint64_t group_occ(const uint4& d, int c, unsigned gmask, unsigned gbase) {
	const uint32_t lo = (c & 1) ? d.z : d.x, hi = (c & 1) ? d.w : d.y;
	const int src = gbase + 6 + (c >> 1);
	const uint32_t rlo = __shfl_sync(gmask, lo, src), rhi = __shfl_sync(gmask, hi, src);
	return (uint64_t)rlo | ((uint64_t)rhi << 32);
}
// BWT[off] of the side (off in 0..383)
__device__ __forceinline__ int group_char(const uint4& d, uint32_t off, unsigned gmask, unsigned gbase) {
	const uint32_t w = sel_word(d, (off >> 4) & 3);
	const uint32_t ch = (w >> ((off & 15) * 2)) & 3;
	return (int)__shfl_sync(gmask, ch, gbase + (off >> 6));
}

}  // namespace cfb
#endif
