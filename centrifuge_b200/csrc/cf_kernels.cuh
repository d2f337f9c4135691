// cf_kernels.cuh -- shared declarations of the sm_90a kernels of the classification path (cfb200.cu).
//
// Work decomposition (one batch of units = reads or pairs), DESIGN.md section 4:
//   k_pack       reads (1 byte/base) -> 2-bit strands in search order + N masks
//   k_search_t   FM-index backward search, the hot loop: ONE THREAD per (unit, mate, strand) greedy walk over the
//                re-cut device index (rank16: one 16-byte gather per rank query; K-mer (with its death bitmap) and walk8 tables
//                delete dependent gathers); one fetch point per loop iteration for all 32 walks of a warp
//   k_search_long  reads over 320 bases: one thread per walk runs the strand's whole search on rank16 (search_strand_dev)
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

static const int kSearchThreads = 128; // 4 warps = 16 walks per CTA

}  // namespace cfb
#endif
