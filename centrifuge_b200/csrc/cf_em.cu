// cf_em.cu -- abundance EM (SQUAREM-accelerated) on the device, SURVEY.md 8f rank 3.
//
// Replaces the iteration of SpeciesMetrics::calculateAbundance (aln_sink.h:274-495, EM step :196-272) for large
// tie-set tables.  The report prints the result with operator<<(double), so the bar is bit-identical doubles;
// IEEE addition is not associative, hence every accumulator is fed in exactly the order the reference's loops
// feed it:
//   psum[k]  one thread per key, its contributions in key order                     (reference: inner loop 1)
//   pn[j]    one thread per species, over its incidence list sorted by (key, position): the order in which the
//            reference's key loop reaches pn[j]                                       (reference: inner loop 2)
//   sums over species (normalisation, ssr, ssv, diff): terms by all threads, then one thread adds them in ascending index order
// and every multiply/add/divide is issued through the _rn intrinsics so that nothing is contracted into an FMA.
// The host (cf_host.cpp) flattens `observed` and computes the start vector; only the iteration runs here.
#include "../../include/cfb200.h"
#include "cf_buf.cuh"

#include <cuda_runtime.h>
#include <cstdio>
#include <vector>

namespace {

struct EmArgs {
	uint64_t n, K;
	const uint64_t* count; const uint64_t* key_off; const uint32_t* target;     // keys
	const uint64_t* inc_off; const uint32_t* inc_key;                           // per-species incidence lists
	const uint64_t* len;
	double* psum;
	double* scal;      // [0] sum [1] ssr [2] ssv [3] diff [4] flag: third EM step wanted [5] flag: converged
};

__global__ void k_em_psum(const EmArgs a, const double* p, int guarded) {
	if(guarded && a.scal[4] == 0.0) return;
	const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(k >= a.K) return;
	double s = 0.0;
	for(uint64_t t = a.key_off[k]; t < a.key_off[k + 1]; t++) s = __dadd_rn(s, p[a.target[t]]);
	a.psum[k] = s;
}
__global__ void k_em_scatter(const EmArgs a, const double* p, double* pn, int guarded) {
	if(guarded && a.scal[4] == 0.0) return;
	const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(j >= a.n) return;
	double acc = 0.0; const double pj = p[j];
	for(uint64_t e = a.inc_off[j]; e < a.inc_off[j + 1]; e++) {
		const uint32_t k = a.inc_key[e]; const double ps = a.psum[k];
		if(ps == 0.0) continue;
		acc = __dadd_rn(acc, __dmul_rn((double)a.count[k], __ddiv_rn(pj, ps)));
	}
	pn[j] = acc;
}
// The sums over species must add in ascending index order (IEEE addition is not associative), but only the additions: the
// terms are computed by all threads first, and the one thread that adds them runs a pure chain of dependent DADDs with the
// loads issued eight ahead (20 000 species: ~0.1 ms instead of ~5 ms with the divisions inside the chain).
__device__ __forceinline__ double serial_sum(const double* q, uint64_t n) {
	double s = 0.0; uint64_t i = 0;
	for(; i + 8 <= n; i += 8) {
		const double x0 = q[i], x1 = q[i + 1], x2 = q[i + 2], x3 = q[i + 3], x4 = q[i + 4], x5 = q[i + 5], x6 = q[i + 6], x7 = q[i + 7];
		s = __dadd_rn(s, x0); s = __dadd_rn(s, x1); s = __dadd_rn(s, x2); s = __dadd_rn(s, x3);
		s = __dadd_rn(s, x4); s = __dadd_rn(s, x5); s = __dadd_rn(s, x6); s = __dadd_rn(s, x7);
	}
	for(; i < n; i++) s = __dadd_rn(s, q[i]);
	return s;
}
__global__ void k_em_quot(const EmArgs a, const double* pn, double* q, int guarded) {      // q[i] = pn[i] / len[i]
	if(guarded && a.scal[4] == 0.0) return;
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < a.n) q[i] = __ddiv_rn(pn[i], (double)a.len[i]);
}
__global__ void k_em_sum(const EmArgs a, const double* q, int guarded) {       // one thread: ascending index
	if(guarded && a.scal[4] == 0.0) return;
	a.scal[0] = serial_sum(q, a.n);
}
__global__ void k_em_scale(const EmArgs a, const double* q, double* pn, int guarded) {      // pn[i] = pn[i] / len[i] / sum
	if(guarded && a.scal[4] == 0.0) return;
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < a.n) pn[i] = __ddiv_rn(q[i], a.scal[0]);
}
__global__ void k_em_diffs(const EmArgs a, const double* p, const double* pn, const double* pn2, double* pr, double* pv, double* r2, double* v2) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= a.n) return;
	const double r = __dsub_rn(pn[i], p[i]);
	const double v = __dsub_rn(__dsub_rn(pn2[i], pn[i]), r);
	pr[i] = r; pv[i] = v; r2[i] = __dmul_rn(r, r); v2[i] = __dmul_rn(v, v);
}
__global__ void k_em_norms(const EmArgs a, const double* r2, const double* v2) {     // two warps, one chain each (lane 0)
	if(threadIdx.x == 0) a.scal[1] = serial_sum(r2, a.n);
	else if(threadIdx.x == 32) { const double ssv = serial_sum(v2, a.n); a.scal[2] = ssv; a.scal[4] = ssv > 0.0 ? 1.0 : 0.0; }
}
__global__ void k_em_extrapolate(const EmArgs a, const double* p, const double* pr, const double* pv, double* pn2) {
	if(a.scal[4] == 0.0) return;
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= a.n) return;
	const double g = -__dsqrt_rn(__ddiv_rn(a.scal[1], a.scal[2]));
	const double x = __dadd_rn(__dsub_rn(p[i], __dmul_rn(__dmul_rn(2.0, g), pr[i])), __dmul_rn(__dmul_rn(g, g), pv[i]));
	pn2[i] = (0.0 < x) ? x : 0.0;                                                    // std::max(0.0, x)
}
__global__ void k_em_absdiff(const EmArgs a, const double* p, const double* pn, double* q) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if(i < a.n) q[i] = p[i] > pn[i] ? __dsub_rn(p[i], pn[i]) : __dsub_rn(pn[i], p[i]);
}
__global__ void k_em_converged(const EmArgs a, const double* q) {   // one thread
	const double d = serial_sum(q, a.n);
	a.scal[3] = d; a.scal[5] = d < 0.0000000001 ? 1.0 : 0.0;
}

static thread_local char g_em_err[256] = "";

}  // namespace

extern "C" const char* cfb_em_last_error(void) { return g_em_err; }

extern "C" int cfb_em_abundance(int device, uint64_t n, uint64_t K, const uint64_t* count, const uint64_t* key_off, const uint32_t* target,
                                const uint64_t* len, double* p, uint64_t* iters, double* last_diff) {
	if(!count || !key_off || !target || !len || !p || !iters || !last_diff || n == 0 || n >= (1ull << 32) || K >= (1ull << 32)) return CFB_EINVAL;
	#define EK(call) do { cudaError_t e_ = (call); if(e_ != cudaSuccess) { snprintf(g_em_err, sizeof g_em_err, "%s failed: %s", #call, cudaGetErrorString(e_)); return CFB_ECUDA; } } while(0)
	EK(cudaSetDevice(device));
	const uint64_t T = key_off[K];
	// incidence lists: species j <- the keys that reach it, in (key, position) order (counting sort keeps it)
	std::vector<uint64_t> inc_off(n + 1, 0); std::vector<uint32_t> inc_key(T);
	for(uint64_t t = 0; t < T; t++) inc_off[target[t] + 1]++;
	for(uint64_t j = 0; j < n; j++) inc_off[j + 1] += inc_off[j];
	{ std::vector<uint64_t> fill(inc_off.begin(), inc_off.end() - 1);
	  for(uint64_t k = 0; k < K; k++) for(uint64_t t = key_off[k]; t < key_off[k + 1]; t++) inc_key[fill[target[t]]++] = (uint32_t)k; }
	auto up = [&](const void* src, size_t bytes, DBuf<uint8_t>& dst) -> cudaError_t {
		cudaError_t e = dst.alloc(bytes ? bytes : 8); if(e != cudaSuccess) return e;
		return bytes ? cudaMemcpy(dst.p, src, bytes, cudaMemcpyHostToDevice) : cudaSuccess;
	};
	EmArgs a; a.n = n; a.K = K;
	DBuf<uint8_t> d_count, d_koff, d_tgt, d_ioff, d_ikey, d_len, d_p; DBuf<double> d_psum, d_scal, d_pn, d_pn2, d_pr, d_pv, d_q, d_q2;
	EK(up(count, K * 8, d_count)); EK(up(key_off, (K + 1) * 8, d_koff)); EK(up(target, T * 4, d_tgt));
	EK(up(inc_off.data(), (n + 1) * 8, d_ioff)); EK(up(inc_key.data(), T * 4, d_ikey)); EK(up(len, n * 8, d_len));
	EK(d_psum.alloc(K + 1));
	EK(d_scal.alloc(8)); EK(cudaMemset(d_scal.p, 0, 64));
	EK(up(p, n * 8, d_p));
	EK(d_pn.alloc(n)); EK(d_pn2.alloc(n));
	EK(d_pr.alloc(n)); EK(d_pv.alloc(n));
	EK(d_q.alloc(n)); EK(d_q2.alloc(n));
	a.count = (const uint64_t*)d_count.p; a.key_off = (const uint64_t*)d_koff.p; a.target = (const uint32_t*)d_tgt.p;
	a.inc_off = (const uint64_t*)d_ioff.p; a.inc_key = (const uint32_t*)d_ikey.p; a.len = (const uint64_t*)d_len.p;
	a.psum = d_psum.p; a.scal = d_scal.p;
	double *P = (double*)d_p.p, *PN = d_pn.p, *PN2 = d_pn2.p, *PR = d_pr.p, *PV = d_pv.p, *Q = d_q.p, *Q2 = d_q2.p;
	const unsigned bk = (unsigned)((K + 255) / 256), bn = (unsigned)((n + 255) / 256);
	auto em_step = [&](const double* src, double* dst, int guarded) {
		if(bk) k_em_psum<<<bk, 256>>>(a, src, guarded);
		k_em_scatter<<<bn, 256>>>(a, src, dst, guarded);
		k_em_quot<<<bn, 256>>>(a, dst, Q, guarded);
		k_em_sum<<<1, 1>>>(a, Q, guarded);
		k_em_scale<<<bn, 256>>>(a, Q, dst, guarded);
	};
	uint64_t it = 0; double sc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	for(;;) {
		em_step(P, PN, 0);
		em_step(PN, PN2, 0);
		k_em_diffs<<<bn, 256>>>(a, P, PN, PN2, PR, PV, Q, Q2);
		k_em_norms<<<1, 64>>>(a, Q, Q2);
		k_em_extrapolate<<<bn, 256>>>(a, P, PR, PV, PN2);
		em_step(PN2, PN, 1);
		k_em_absdiff<<<bn, 256>>>(a, P, PN, Q);
		k_em_converged<<<1, 1>>>(a, Q);
		EK(cudaMemcpy(sc, d_scal.p, 64, cudaMemcpyDeviceToHost));
		if(sc[5] != 0.0) break;
		if(++it >= 10000) break;
		double* tmp = P; P = PN; PN = tmp;                      // p = pn
	}
	EK(cudaMemcpy(p, P, n * 8, cudaMemcpyDeviceToHost));
	*iters = it; *last_diff = sc[3];
	#undef EK
	return CFB_OK;
}
