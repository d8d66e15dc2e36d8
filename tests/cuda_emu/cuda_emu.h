// cuda_emu.h -- TEST INFRASTRUCTURE.  A small CUDA execution model on the CPU, enough to run the kernels of
// sharpziplib_b200/csrc (the unmodified sources, preprocessed by build_emu.py) without a GPU: every CUDA thread of a block is
// a fiber (ucontext) with its own stack, blocks run one after the other, the fibers of a block are scheduled cooperatively and
// switch only at barriers and warp collectives.  Deterministic, single OS thread, so atomics are plain operations.
//
// It exists to CHECK kernels (bit-exactness against the oracle, out-of-bounds shared memory, barrier mismatches) when GPU
// time is scarce -- it says nothing about performance.  The product never loads it: tests/cuda_emu/run_emulated.py swaps the
// library inside the test process only.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <ucontext.h>

#include <functional>
#include <vector>

#define __CUDA_ARCH__ 900
#define B200Z_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __shared__ static
#define __constant__
#define __launch_bounds__(...)
#define __align__(n) alignas(n)

struct uint2 { uint32_t x, y; };
struct int2 { int32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct dim3 {
	unsigned x, y, z;
	dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline int2 make_int2(int32_t x, int32_t y) { return int2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

namespace emu {

extern size_t g_stack_bytes; // per CUDA thread; B200Z_EMU_STACK_KB (default 1024; AddressSanitizer clears a context's whole
                              // shadow stack on every switch, so its runs want this small)
constexpr size_t kMaxSmem = 256 * 1024;

struct Warp {
	int live = 0, arrived = 0;
	uint32_t gen = 0;
	uint64_t vals[32];
	uint32_t present = 0, preds = 0;
};
struct Fiber {
	ucontext_t ctx;
	dim3 tid;
	int linear = 0, lane = 0, warp = 0;
	bool done = false;
	void *stack = nullptr;
};
struct Block {
	std::vector<Fiber> fibers;
	std::vector<Warp> warps;
	int live = 0, arrived = 0;
	uint32_t gen = 0;
	int or_acc = 0;
	uint32_t or_reset_gen = 0xFFFFFFFFu;
	int cnt_acc = 0;
	uint32_t cnt_reset_gen = 0xFFFFFFFFu;
	dim3 bid, bdim, gdim;
	uint8_t *smem = nullptr;
	ucontext_t sched;
	std::function<void()> body;
};
extern Block *g_block;
extern Fiber *g_cur;
extern uint64_t g_events; // barrier arrivals and thread exits: a scheduling round without any is a deadlock

inline void yield() { swapcontext(&g_cur->ctx, &g_block->sched); }

inline void block_barrier() {
	Block &b = *g_block;
	const uint32_t gen = b.gen;
	g_events++; // an arrival is progress
	if (++b.arrived >= b.live) {
		b.arrived = 0;
		b.gen++;
	} else {
		while (b.gen == gen) yield();
	}
}
inline void warp_barrier() {
	Warp &w = g_block->warps[g_cur->warp];
	const uint32_t gen = w.gen;
	g_events++;
	if (++w.arrived >= w.live) {
		w.arrived = 0;
		w.gen++;
	} else {
		while (w.gen == gen) yield();
	}
}
// every live lane contributes a value; returns everybody's values and who was there
inline void warp_gather(uint64_t v, uint64_t out[32], uint32_t &present) {
	Warp &w = g_block->warps[g_cur->warp];
	w.vals[g_cur->lane] = v;
	w.present |= 1u << g_cur->lane;
	warp_barrier();
	for (int i = 0; i < 32; i++) out[i] = w.vals[i];
	present = w.present;
	warp_barrier();
	if (g_cur->lane == __builtin_ctz(present)) w.present = 0; // (everybody has read; the next collective starts clean)
	warp_barrier();
}
void launch(dim3 grid, dim3 block, size_t smem_bytes, std::function<void()> body);
inline uint8_t *dyn_smem() { return g_block->smem; }

} // namespace emu

#define threadIdx (emu::g_cur->tid)
#define blockIdx (emu::g_block->bid)
#define blockDim (emu::g_block->bdim)
#define gridDim (emu::g_block->gdim)

static inline void __syncthreads() { emu::block_barrier(); }
static inline int __syncthreads_or(int pred) {
	emu::Block &b = *emu::g_block;
	b.or_acc |= pred ? 1 : 0;
	emu::block_barrier();
	const int r = b.or_acc; // everybody has contributed
	emu::block_barrier();   // everybody has read
	if (b.or_reset_gen != b.gen) { // the first thread to get here clears the accumulator for the next use
		b.or_acc = 0;
		b.or_reset_gen = b.gen;
	}
	return r;
}
static inline int __syncthreads_count(int pred) {
	emu::Block &b = *emu::g_block;
	b.cnt_acc += pred ? 1 : 0;
	emu::block_barrier();
	const int r = b.cnt_acc; // everybody has contributed
	emu::block_barrier();    // everybody has read
	if (b.cnt_reset_gen != b.gen) {
		b.cnt_acc = 0;
		b.cnt_reset_gen = b.gen;
	}
	return r;
}
static inline void __syncwarp(uint32_t = 0xffffffffu) { emu::warp_barrier(); }

template <class T> static inline uint64_t emu_bits(T v) {
	static_assert(sizeof(T) <= 8, "");
	uint64_t u = 0;
	memcpy(&u, &v, sizeof(T));
	return u;
}
template <class T> static inline T emu_unbits(uint64_t u) {
	T v;
	memcpy(&v, &u, sizeof(T));
	return v;
}
template <class T> static inline T __shfl_sync(uint32_t, T v, int src, int width = 32) {
	uint64_t a[32];
	uint32_t pr;
	emu::warp_gather(emu_bits(v), a, pr);
	(void)width;
	return emu_unbits<T>(a[src & 31]);
}
template <class T> static inline T __shfl_up_sync(uint32_t, T v, unsigned d) {
	uint64_t a[32];
	uint32_t pr;
	emu::warp_gather(emu_bits(v), a, pr);
	const int l = emu::g_cur->lane;
	return l >= (int)d ? emu_unbits<T>(a[l - (int)d]) : v;
}
template <class T> static inline T __shfl_down_sync(uint32_t, T v, unsigned d) {
	uint64_t a[32];
	uint32_t pr;
	emu::warp_gather(emu_bits(v), a, pr);
	const int l = emu::g_cur->lane;
	return l + (int)d < 32 ? emu_unbits<T>(a[l + (int)d]) : v;
}
template <class T> static inline T __shfl_xor_sync(uint32_t, T v, int m) {
	uint64_t a[32];
	uint32_t pr;
	emu::warp_gather(emu_bits(v), a, pr);
	return emu_unbits<T>(a[(emu::g_cur->lane ^ m) & 31]);
}
static inline uint32_t __ballot_sync(uint32_t, int pred) {
	uint64_t a[32];
	uint32_t pr, r = 0;
	emu::warp_gather(pred ? 1 : 0, a, pr);
	for (int i = 0; i < 32; i++)
		if ((pr >> i & 1) && a[i]) r |= 1u << i;
	return r;
}
static inline int __any_sync(uint32_t m, int pred) { return __ballot_sync(m, pred) != 0; }
static inline int __all_sync(uint32_t m, int pred) {
	uint64_t a[32];
	uint32_t pr;
	emu::warp_gather(pred ? 1 : 0, a, pr);
	(void)m;
	for (int i = 0; i < 32; i++)
		if ((pr >> i & 1) && !a[i]) return 0;
	return 1;
}
template <class T> static inline uint32_t __match_any_sync(uint32_t, T v) {
	uint64_t a[32];
	uint32_t pr, r = 0;
	emu::warp_gather(emu_bits(v), a, pr);
	for (int i = 0; i < 32; i++)
		if ((pr >> i & 1) && a[i] == emu_bits(v)) r |= 1u << i;
	return r;
}

template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31)); }
static inline uint32_t __funnelshift_l(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)(((((uint64_t)hi << 32) | lo) << (sh & 31)) >> 32); }
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) { // PRMT, default mode: selector nibble k picks byte k of (b:a)
	const uint64_t v = ((uint64_t)b << 32) | a;
	uint32_t r = 0;
	for (int k = 0; k < 4; k++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * k)) & 7))) & 0xFF) << (8 * k);
	return r;
}
static inline int __ffs(int x) { return x ? __builtin_ctz((unsigned)x) + 1 : 0; }
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline uint32_t __brev(uint32_t x) {
	uint32_t r = 0;
	for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i);
	return r;
}
template <class T> static inline T atomicAdd(T *p, T v) { T o = *p; *p = (T)(o + v); return o; }
template <class T> static inline T atomicOr(T *p, T v) { T o = *p; *p = (T)(o | v); return o; }
template <class T> static inline T atomicMin(T *p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicMax(T *p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicXor(T *p, T v) { T o = *p; *p = (T)(o ^ v); return o; }
static inline void __pipeline_memcpy_async(void *dst, const void *src, size_t n) { memcpy(dst, src, n); }
static inline void __pipeline_commit() {}
static inline void __pipeline_wait_prior(int) {}

// ---- the slice of the CUDA runtime the library's host code uses: "device" memory is host memory ----
typedef int cudaError_t;
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyHostToHost };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9, cudaHostAllocDefault = 0 };
static inline const char *cudaGetErrorString(cudaError_t e) { return e ? "emulated CUDA error" : "no error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) {
	void *q = nullptr;
	if (posix_memalign(&q, 256, n ? n : 256)) return cudaErrorMemoryAllocation;
	static const int fill = getenv("B200Z_EMU_FILL") ? atoi(getenv("B200Z_EMU_FILL")) : 0xCD; // B200Z_EMU_FILL=0: what a fresh device usually holds
	if (fill < 0) { // B200Z_EMU_FILL=-<seed>: pseudo-random bytes, words of 0xFFFFFFFF sprinkled in (what other processes leave behind)
		static uint64_t st = (uint64_t)(-fill) * 0x9E3779B97F4A7C15ull + 1;
		uint32_t *w = (uint32_t *)q;
		for (size_t i = 0; i < n / 4; i++) {
			st = st * 6364136223846793005ull + 1442695040888963407ull;
			const uint32_t r = (uint32_t)(st >> 32);
			w[i] = (r & 7u) == 0 ? 0xFFFFFFFFu : (r & 7u) == 1 ? 0xFFFFFFFEu : r;
		}
	} else
	memset(q, fill, n); // cudaMalloc does not clear either: make reads of unwritten memory visible
	*p = (T *)q;
	return cudaSuccess;
}
template <class T> static inline cudaError_t cudaMallocAsync(T **p, size_t n, cudaStream_t) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaFreeAsync(void *p, cudaStream_t) { free(p); return cudaSuccess; }
template <class T> static inline cudaError_t cudaHostAlloc(T **p, size_t n, unsigned) { return cudaMalloc(p, n); }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = nullptr; return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2 };
struct cudaPointerAttributes { cudaMemoryType type; };
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *) { a->type = cudaMemoryTypeUnregistered; return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = nullptr; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
enum { cudaDevAttrMultiProcessorCount = 16 };
static inline cudaError_t cudaDeviceGetAttribute(int *v, int, int) { *v = 2; return cudaSuccess; } // "two SMs"
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) { *n = 2; return cudaSuccess; }
#define cudaMemcpyToSymbol(sym, src, n, ...) (memcpy((void *)&(sym), (src), (n)), cudaSuccess)

// kernel<<<grid, block, smem, stream>>>(args...) is rewritten by build_emu.py into this
#define EMU_LAUNCH(kernel, grid, block, smem, ...) emu::launch(dim3(grid), dim3(block), (size_t)(smem), [=]() { kernel(__VA_ARGS__); })
