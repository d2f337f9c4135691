// tests/native/gunzip_host.cpp -- TEST ONLY.  Compiles the device inflater's per-chunk decode code
// (centrifuge_b200/csrc/cf_inflate.h) for the host, so that tests/test_gunzip_host.py can check it against zlib
// without a GPU.  This is not a CPU fallback: nothing in the product links or loads this file.
#include <vector>
#include "../../centrifuge_b200/csrc/cf_inflate.h"

extern "C" {

// res: {status, n_sym, end_bit, end_hdr, safe_bit, safe_hdr, safe_sym, first_type}
void gzh_inflate_chunk(const uint8_t* in, uint64_t n, uint64_t start_bit, uint64_t start_hdr, uint64_t stop_bit,
                       uint16_t* out, uint32_t cap, int64_t* res) {
	static cfz::Tables t;
	cfz::ChunkResult r;
	cfz::inflate_chunk(in, n, start_bit, start_hdr, stop_bit, out, cap, t, r);
	res[0] = r.status; res[1] = r.n_sym; res[2] = (int64_t)r.end_bit; res[3] = (int64_t)r.end_hdr;
	res[4] = (int64_t)r.safe_bit; res[5] = (int64_t)r.safe_hdr; res[6] = r.safe_sym; res[7] = r.first_type;
}

// every bit offset in [from, to) whose block header looks valid (verified: whose whole block does too); returns how
// many (at most cap are stored)
uint64_t gzh_scan(const uint8_t* in, uint64_t n, uint64_t from, uint64_t to, uint64_t* out, uint64_t cap, int verified) {
	static cfz::Tables t;
	uint64_t k = 0;
	for(uint64_t b = from; b < to; b++)
		if(verified ? cfz::block_start_verified(in, n, b, t) : cfz::block_header_plausible(in, n, b, t)) { if(k < cap) out[k] = b; k++; }
	return k;
}

}
