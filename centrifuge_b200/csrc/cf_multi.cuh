// cf_multi.cuh -- what a multi-GPU run needs from the library (SURVEY.md 8e), plus the measurement hooks of bench.py.
// Included at the end of cfb200.cu.
//
//   * per-taxon counters: reading / resetting the context's device-side counters (CountsCtx in cfb200.cu)
//   * the one collective of the path: ncclAllReduce(ncclUint64, ncclSum) of those counters over the ranks
//     (replaces the dense part of SpeciesMetrics::merge, aln_sink.h:109-140: per-thread metrics summed at the end of
//     the run, centrifuge.cpp:3175-3179); the sparse `observed` tie sets are merged on the host as the reference does
//   * the random-gather ceiling of the device over the replica's own arrays (the denominator of the walk kernel's
//     roofline, measured in the same process and on the same footprint as the kernel it bounds)
//
// NCCL is resolved at run time (dlopen "libnccl.so.2"): a process that already holds a copy -- torch's bundled one under
// torchrun -- keeps using that copy, and single-GPU users never load it.
#include <dlfcn.h>
#include <nccl.h>

// ------------------------------------------------------------------------------ counters
extern "C" int cfb_ctx_count_records(cfb_ctx* c, int on) {
	if(!c) return fail(CFB_EINVAL, "null ctx");
	CK(cudaSetDevice(c->ix->device));
	if(on) { int rc = counts_init(c); if(rc) return rc; }
	c->fold_records = on != 0;
	return CFB_OK;
}
extern "C" int cfb_counts_taxids(cfb_ctx* c, uint64_t* taxid, uint64_t cap, uint64_t* n) {
	if(!c || !n) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	int rc = counts_init(c); if(rc) return rc;
	*n = c->cnt.n;
	if(taxid) { if(cap < c->cnt.n) return fail(CFB_EINVAL, "cfb_counts_taxids: buffer too small"); memcpy(taxid, c->cnt.h_taxid.data(), (size_t)c->cnt.n * 8); }
	return CFB_OK;
}
extern "C" int cfb_counts_reset(cfb_ctx* c) {
	if(!c) return fail(CFB_EINVAL, "null ctx");
	CK(cudaSetDevice(c->ix->device));
	if(!c->cnt.ready) return CFB_OK;
	CK(cudaDeviceSynchronize());
	CK(cudaMemset(c->cnt.total.p, 0, 3ull * c->cnt.n * 8)); CK(cudaMemset(c->cnt.global.p, 0, 3ull * c->cnt.n * 8));
	c->cnt.reduced = false;
	return CFB_OK;
}
extern "C" int cfb_counts_dense(cfb_ctx* c, int global, uint64_t* out, uint64_t cap) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	int rc = counts_init(c); if(rc) return rc;
	if(cap < 3ull * c->cnt.n) return fail(CFB_EINVAL, "cfb_counts_dense: buffer too small");
	if(global && !c->cnt.reduced) return fail(CFB_EINVAL, "no reduced counters: call cfb_counts_allreduce first");
	CK(cudaDeviceSynchronize());
	CK(cudaMemcpy(out, global ? c->cnt.global.p : c->cnt.total.p, 3ull * c->cnt.n * 8, cudaMemcpyDeviceToHost));
	return CFB_OK;
}
extern "C" int cfb_counts_read(cfb_ctx* c, int global, uint64_t* taxid, uint64_t* n_reads, uint64_t* n_unique, uint64_t* n_obs1, uint64_t cap, uint64_t* n) {
	if(!c || !n) return fail(CFB_EINVAL, "null argument");
	*n = 0;
	if(!c->cnt.ready) return CFB_OK;
	const size_t nsp = c->cnt.n;
	std::vector<uint64_t> h(3 * nsp);
	int rc = cfb_counts_dense(c, global, h.data(), h.size()); if(rc) return rc;
	uint64_t k = 0;
	for(size_t i = 0; i < nsp; i++) if(h[i]) {
		if(k < cap && taxid && n_reads && n_unique && n_obs1) { taxid[k] = c->cnt.h_taxid[i]; n_reads[k] = h[i]; n_unique[k] = h[nsp + i]; n_obs1[k] = h[2 * nsp + i]; }
		k++;
	}
	*n = k;
	return CFB_OK;
}

// ------------------------------------------------------------------------------ NCCL
namespace {
struct NcclApi {
	void* lib = nullptr; bool tried = false; std::string err;
	ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*GroupStart)() = nullptr;
	ncclResult_t (*GroupEnd)() = nullptr;
	const char* (*GetErrorString)(ncclResult_t) = nullptr;
	ncclResult_t (*GetVersion)(int*) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;
bool nccl_load() {
	std::lock_guard<std::mutex> l(g_nccl_mu);
	NcclApi& n = g_nccl;
	if(n.tried) return n.lib != nullptr;
	n.tried = true;
	const char* names[] = {getenv("CFB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
	for(const char* nm : names) { if(nm && *nm) { n.lib = dlopen(nm, RTLD_NOW | RTLD_LOCAL); if(n.lib) break; const char* e = dlerror(); n.err = e ? e : "dlopen failed"; } }
	if(!n.lib) return false;
	#define SYM(field, name) do { *(void**)(&n.field) = dlsym(n.lib, name); if(!n.field) { n.err = std::string("missing symbol ") + name; dlclose(n.lib); n.lib = nullptr; return false; } } while(0)
	SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommInitAll, "ncclCommInitAll"); SYM(CommDestroy, "ncclCommDestroy");
	SYM(AllReduce, "ncclAllReduce"); SYM(GroupStart, "ncclGroupStart"); SYM(GroupEnd, "ncclGroupEnd"); SYM(GetErrorString, "ncclGetErrorString"); SYM(GetVersion, "ncclGetVersion");
	#undef SYM
	return true;
}
}  // namespace
#define NK(call) do { ncclResult_t r_ = (call); if(r_ != ncclSuccess) return fail(CFB_ECUDA, "%s failed: %s", #call, g_nccl.GetErrorString(r_)); } while(0)

static int comm_prepare(cfb_ctx* c) {
	CK(cudaSetDevice(c->ix->device));
	int rc = counts_init(c); if(rc) return rc;
	if(!c->comm_st) CK(c->comm_st.create());
	return CFB_OK;
}
static_assert(sizeof(ncclUniqueId) == CFB_COMM_ID_BYTES, "ncclUniqueId size");

extern "C" int cfb_comm_unique_id(uint8_t id[CFB_COMM_ID_BYTES]) {
	if(!id) return fail(CFB_EINVAL, "null argument");
	if(!nccl_load()) return fail(CFB_ENODEV, "NCCL is not available: %s", g_nccl.err.c_str());
	ncclUniqueId u; NK(g_nccl.GetUniqueId(&u));
	memcpy(id, &u, sizeof u);
	return CFB_OK;
}
extern "C" int cfb_comm_init_rank(cfb_ctx* c, int nranks, int rank, const uint8_t id[CFB_COMM_ID_BYTES]) {
	if(!c || !id || nranks < 1 || rank < 0 || rank >= nranks) return fail(CFB_EINVAL, "cfb_comm_init_rank: bad argument");
	if(c->comm) return fail(CFB_EINVAL, "context already belongs to a communicator");
	if(!nccl_load()) return fail(CFB_ENODEV, "NCCL is not available: %s", g_nccl.err.c_str());
	int rc = comm_prepare(c); if(rc) return rc;
	ncclUniqueId u; memcpy(&u, id, sizeof u);
	ncclComm_t comm = nullptr;
	NK(g_nccl.CommInitRank(&comm, nranks, u, rank));
	c->comm = comm; c->comm_rank = rank; c->comm_size = nranks;
	return CFB_OK;
}
extern "C" int cfb_comm_init_all(cfb_ctx* const* ctxs, int n) {
	if(!ctxs || n < 1 || n > 64) return fail(CFB_EINVAL, "cfb_comm_init_all: bad argument");
	for(int i = 0; i < n; i++) { if(!ctxs[i] || ctxs[i]->comm) return fail(CFB_EINVAL, "cfb_comm_init_all: null context or context already in a communicator"); }
	for(int i = 0; i < n; i++) for(int j = 0; j < i; j++) if(ctxs[i]->ix->device == ctxs[j]->ix->device) return fail(CFB_EINVAL, "cfb_comm_init_all: two contexts on device %d", ctxs[i]->ix->device);
	if(!nccl_load()) return fail(CFB_ENODEV, "NCCL is not available: %s", g_nccl.err.c_str());
	std::vector<int> devs(n); std::vector<ncclComm_t> comms(n, nullptr);
	for(int i = 0; i < n; i++) { int rc = comm_prepare(ctxs[i]); if(rc) return rc; devs[i] = ctxs[i]->ix->device; }
	NK(g_nccl.CommInitAll(comms.data(), n, devs.data()));
	for(int i = 0; i < n; i++) { ctxs[i]->comm = comms[i]; ctxs[i]->comm_rank = i; ctxs[i]->comm_size = n; }
	return CFB_OK;
}

// Sum the per-taxon counters of every rank: `ctxs` are this process's contexts (one under torchrun / MPI, all of them in
// a single-process multi-GPU run); every rank of the communicator must call it.  Afterwards cfb_counts_read/dense
// (global = 1) return the totals on every rank.  Without a communicator (one GPU) the totals are the local ones.
extern "C" int cfb_counts_allreduce(cfb_ctx* const* ctxs, int n, uint64_t* dense_out, uint64_t cap) {
	if(!ctxs || n < 1) return fail(CFB_EINVAL, "cfb_counts_allreduce: bad argument");
	for(int i = 0; i < n; i++) {
		cfb_ctx* c = ctxs[i];
		if(!c) return fail(CFB_EINVAL, "null context");
		int rc = comm_prepare(c); if(rc) return rc;
		// every collected batch has queued the commit of its counters on its slot's stream: order the collective behind
		// those commits on the device, without draining batches that are still in flight
		for(int k = 0; k < kSlots; k++) { Slot& s = c->slots[k]; if(s.commit_pending) { CK(cudaStreamWaitEvent(c->comm_st, s.ev[5], 0)); s.commit_pending = false; } }
	}
	bool any_comm = false;
	for(int i = 0; i < n; i++) any_comm |= ctxs[i]->comm != nullptr;
	if(n > 1 && !any_comm) return fail(CFB_EINVAL, "cfb_counts_allreduce: %d contexts without a communicator (call cfb_comm_init_all)", n);
	const bool grouped = n > 1;
	if(grouped) NK(g_nccl.GroupStart());
	for(int i = 0; i < n; i++) {
		cfb_ctx* c = ctxs[i];
		CK(cudaSetDevice(c->ix->device));
		const size_t cnt = 3ull * c->cnt.n;
		if(c->comm) NK(g_nccl.AllReduce(c->cnt.total.p, c->cnt.global.p, cnt, ncclUint64, ncclSum, (ncclComm_t)c->comm, c->comm_st));
		else CK(cudaMemcpyAsync(c->cnt.global.p, c->cnt.total.p, cnt * 8, cudaMemcpyDeviceToDevice, c->comm_st));
	}
	if(grouped) NK(g_nccl.GroupEnd());
	for(int i = 0; i < n; i++) { cfb_ctx* c = ctxs[i]; CK(cudaSetDevice(c->ix->device)); CK(cudaStreamSynchronize(c->comm_st)); c->cnt.reduced = true; }
	if(dense_out) return cfb_counts_dense(ctxs[0], 1, dense_out, cap);
	return CFB_OK;
}
extern "C" int cfb_comm_info(const cfb_ctx* c, int* rank, int* size, int* nccl_version) {
	if(!c) return fail(CFB_EINVAL, "null ctx");
	if(rank) *rank = c->comm_rank; if(size) *size = c->comm ? c->comm_size : 1;
	if(nccl_version) { *nccl_version = 0; if(g_nccl.lib) g_nccl.GetVersion(nccl_version); }
	return CFB_OK;
}

// ------------------------------------------------------------------------------ measurement hooks
extern "C" int cfb_ctx_requests(cfb_ctx* c, uint64_t out[5]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	Counters h; CK(cudaMemcpy(&h, c->d_ctr.p, sizeof h, cudaMemcpyDeviceToHost));
	out[0] = h.req_rank16; out[1] = h.req_ftab2; out[2] = h.req_ftabk; out[3] = h.req_walk8; out[4] = h.req_ftabd;
	return CFB_OK;
}
extern "C" int cfb_ctx_request_breakdown(cfb_ctx* c, uint64_t out[8]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	Counters h; CK(cudaMemcpy(&h, c->d_ctr.p, sizeof h, cudaMemcpyDeviceToHost));
	out[0] = h.r16_w1; out[1] = h.r16_w2_4; out[2] = h.r16_w5;
	out[3] = h.w8_try_row; out[4] = h.w8_ok_row; out[5] = h.w8_try_range; out[6] = h.w8_ok_range; out[7] = h.w8_ok_w5;
	return CFB_OK;
}
extern "C" int cfb_ctx_search_iter_stats(cfb_ctx* c, uint64_t out[8]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	Counters h; CK(cudaMemcpy(&h, c->d_ctr.p, sizeof h, cudaMemcpyDeviceToHost));
	out[0] = h.it_warp; out[1] = h.it_lane_req; out[2] = h.it_consumers; out[3] = h.it_restarts; out[4] = h.it_task;
	out[5] = h.clk_head; out[6] = h.clk_wait; out[7] = h.clk_tail;
	return CFB_OK;
}
extern "C" int cfb_ctx_score_stats(cfb_ctx* c, uint64_t out[23]) {
	if(!c || !out) return fail(CFB_EINVAL, "null argument");
	CK(cudaSetDevice(c->ix->device));
	Counters h; CK(cudaMemcpy(&h, c->d_ctr.p, sizeof h, cudaMemcpyDeviceToHost));
	out[0] = h.sc_units; out[1] = h.sc_rows; out[2] = h.sc_nmap; out[3] = h.sc_reduce; out[4] = h.sc_rounds; out[5] = h.sc_warps; out[6] = h.sc_warps_global;
	for(int i = 0; i < 8; i++) { out[7 + i] = h.sc_rows_hist[i]; out[15 + i] = h.sc_nmap_hist[i]; }
	return CFB_OK;
}

__device__ __forceinline__ uint64_t gmix(uint64_t x) { x += 0x9E3779B97F4A7C15ull; x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull; x = (x ^ (x >> 27)) * 0x94D049BB133111EBull; return x ^ (x >> 31); }
// independent, uniformly random gathers of W 8-byte words per request from array `a` of `n` requests' worth, `iters` x ILP per thread
template <int W, int ILP>
__global__ void __launch_bounds__(128) k_gather_probe(const unsigned long long* __restrict__ a, uint64_t n, uint32_t iters, unsigned long long* sink) {
	const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	uint64_t h = gmix(tid * 0x2545F4914F6CDD1Dull + 1), acc = 0;
	for(uint32_t it = 0; it < iters; it++) {
		unsigned long long v[ILP][W];
		#pragma unroll
		for(int k = 0; k < ILP; k++) {
			h = gmix(h + k);
			const uint64_t u = h % n;
			if(W == 2) { const ulonglong2 q = __ldg(reinterpret_cast<const ulonglong2*>(a) + u); v[k][0] = q.x; v[k][W - 1] = q.y; }
			else v[k][0] = __ldg(a + u);
		}
		#pragma unroll
		for(int k = 0; k < ILP; k++) acc += W == 2 ? (v[k][0] ^ (v[k][W - 1] << 1)) : v[k][0];
	}
	if(acc == 0x123456789abcull) *sink = acc;
}
// table: 0 = the loaded rank structure, rank16 or the compact layout (16-byte pieces), 1 = K-mer jump table (16-byte), 2 = walk8 (8-byte), 3 = resolve table (8-byte words of it),
// 4 = death bits, which have no table of their own (always "not built")
// ctas_per_sm CTAs of 128 threads per SM (all resident when <= 16), ilp independent requests per thread in flight
extern "C" int cfb_gather_rate(const cfb_index* ix, int table, uint64_t n_requests, int ctas_per_sm, int ilp, double* g_requests_per_s, double* ms_out) {
	if(!ix || !g_requests_per_s || ix->device < 0 || ctas_per_sm < 1 || (ilp != 1 && ilp != 2 && ilp != 4)) return fail(CFB_EINVAL, "cfb_gather_rate: bad argument");
	CK(cudaSetDevice(ix->device));
	const cfb_index_tables& t = ix->tables; const IndexView& v = ix->view;
	const unsigned long long* base = nullptr; uint64_t n = 0; int W = 1;
	switch(table) {
		case 0: base = (const unsigned long long*)(v.cr ? v.cr : v.rank16); n = (v.cr ? t.sides_bytes : t.rank16_bytes) / 16; W = 2; break;
		case 1: base = (const unsigned long long*)v.ftabk; n = t.ftabk_bytes / 16; W = 2; break;
		case 2: base = (const unsigned long long*)v.walk8; n = t.walk8_bytes / 8; W = 1; break;
		case 3: base = v.rtab32 ? (const unsigned long long*)v.rtab32 : (const unsigned long long*)v.rtab16; n = t.resolve_table_bytes / 8; W = 1; break;
		case 4: break;      // death bits: no table of their own, they live in the K-mer table's entries
		default: return fail(CFB_EINVAL, "cfb_gather_rate: unknown table %d", table);
	}
	if(!base || n == 0) return fail(CFB_EINVAL, "cfb_gather_rate: table %d is not built", table);
	const int threads = 128;
	const int blocks = ix->sm_count * ctas_per_sm;
	const uint64_t per_iter = (uint64_t)blocks * threads * ilp;
	const uint32_t iters = (uint32_t)std::max<uint64_t>(1, n_requests / per_iter);
	DBuf<unsigned long long> sink; CK(sink.alloc(1));
	Event e0, e1; CK(e0.create()); CK(e1.create());
	auto launch = [&](uint32_t it) {
		if(W == 2) { if(ilp == 4) k_gather_probe<2, 4><<<blocks, threads>>>(base, n, it, sink.p); else if(ilp == 2) k_gather_probe<2, 2><<<blocks, threads>>>(base, n, it, sink.p); else k_gather_probe<2, 1><<<blocks, threads>>>(base, n, it, sink.p); }
		else { if(ilp == 4) k_gather_probe<1, 4><<<blocks, threads>>>(base, n, it, sink.p); else if(ilp == 2) k_gather_probe<1, 2><<<blocks, threads>>>(base, n, it, sink.p); else k_gather_probe<1, 1><<<blocks, threads>>>(base, n, it, sink.p); }
	};
	launch(std::max<uint32_t>(1, iters / 16)); CK(cudaDeviceSynchronize());      // warm-up
	CK(cudaEventRecord(e0)); launch(iters); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
	float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
	CK(cudaGetLastError());
	*g_requests_per_s = (double)per_iter * iters / ((double)ms * 1e6);
	if(ms_out) *ms_out = ms;
	return CFB_OK;
}
// the ceiling: 16 CTAs per SM x 4 requests per thread = 8192 requests in flight per SM
extern "C" int cfb_gather_ceiling(const cfb_index* ix, int table, uint64_t n_requests, double* g_requests_per_s, double* ms_out) {
	return cfb_gather_rate(ix, table, n_requests, 16, 4, g_requests_per_s, ms_out);
}
