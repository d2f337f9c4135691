// cf_buf.cuh -- the owners of every device allocation, pinned host buffer, stream and event of the library.
//
// Each type frees what it holds when it goes, so an object releases its resources by being destroyed and a half-built one
// by going out of scope.  An object whose kernels or copies may still be in flight when it goes (a context, a decoder)
// synchronises its streams in its destructor body, which runs before any member is freed.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <utility>

// A device (Host = false) or pinned host (Host = true) array of T.  Pinned memory is portable: several contexts on
// different devices may DMA from the same buffer.
template <class T, bool Host> struct Buf {
	T* p = nullptr; size_t cap = 0;
	Buf() = default;
	Buf(Buf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, size_t(0))) {}
	Buf& operator=(Buf&& o) noexcept { if(this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, size_t(0)); } return *this; }
	~Buf() { release(); }
	// grow-only with an eighth of slack, for arrays that follow the batch size
	cudaError_t ensure(size_t n) { return n <= cap ? cudaSuccess : alloc(n + n / 8 + 16); }
	// grow-only, exactly n
	cudaError_t ensure_exact(size_t n) { return n <= cap ? cudaSuccess : alloc(n); }
	// free, then exactly max(n, 1)
	cudaError_t alloc(size_t n) {
		release();
		if(n == 0) n = 1;
		const cudaError_t e = Host ? cudaHostAlloc((void**)&p, n * sizeof(T), cudaHostAllocPortable) : cudaMalloc((void**)&p, n * sizeof(T));
		if(e == cudaSuccess) cap = n; else p = nullptr;
		return e;
	}
	void release() {
		if(p) { if(Host) cudaFreeHost(p); else cudaFree(p); }
		p = nullptr; cap = 0;
	}
};
template <class T> using DBuf = Buf<T, false>;
template <class T> using HBuf = Buf<T, true>;

struct Stream {       // a non-blocking stream
	cudaStream_t st = nullptr;
	Stream() = default;
	Stream(Stream&& o) noexcept : st(std::exchange(o.st, nullptr)) {}
	Stream& operator=(Stream&& o) noexcept { std::swap(st, o.st); return *this; }
	~Stream() { if(st) cudaStreamDestroy(st); }
	cudaError_t create() { return cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking); }
	operator cudaStream_t() const { return st; }
};

struct Event {
	cudaEvent_t ev = nullptr;
	Event() = default;
	Event(Event&& o) noexcept : ev(std::exchange(o.ev, nullptr)) {}
	Event& operator=(Event&& o) noexcept { std::swap(ev, o.ev); return *this; }
	~Event() { if(ev) cudaEventDestroy(ev); }
	cudaError_t create(unsigned flags = cudaEventDefault) { return cudaEventCreateWithFlags(&ev, flags); }
	operator cudaEvent_t() const { return ev; }
};

// Page-locked host memory (cfb_host_alloc, HBuf) is DMA'd from where it is; pageable memory is staged through a pinned buffer.
inline bool is_pinned(const void* p) {
	cudaPointerAttributes at;
	if(cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
	return at.type == cudaMemoryTypeHost;
}
