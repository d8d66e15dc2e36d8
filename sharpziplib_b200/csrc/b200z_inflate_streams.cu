// b200z_inflate_streams.cu -- the device side of the inflate carry (b200z_handles.cu): every Inflater stream, a handle's
// or one of a set's, keeps its window (the last 32 KiB of output) in a device window pool between runs, so a run uploads
// only compressed bytes.  k_carry_stage fills a plan's input slots from the pool and one packed upload; k_carry_window
// writes the window behind a run back into the pool.  One CTA per stream.
#include "b200z_internal.cuh"

namespace b200z {

constexpr int kCarryThreads = 256;

// one CTA copies n bytes; 16-byte words where source and destination share their alignment
__device__ __forceinline__ void cta_copy(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, int64_t n) {
	int64_t head = n;
	if (((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15) == 0) {
		head = (int64_t)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15);
		if (head > n) head = n;
		const int64_t nv = (n - head) >> 4;
		uint4 *d = reinterpret_cast<uint4 *>(dst + head);
		const uint4 *s = reinterpret_cast<const uint4 *>(src + head);
		for (int64_t v = threadIdx.x; v < nv; v += blockDim.x) d[v] = s[v];
		for (int64_t b = head + (nv << 4) + threadIdx.x; b < n; b += blockDim.x) dst[b] = src[b];
	}
	for (int64_t b = threadIdx.x; b < head; b += blockDim.x) dst[b] = src[b];
}

// The window of pool slot p is the last win_len bytes of the slot, so it ends on a 16-byte boundary like the slot's
// compressed bytes do: the dictionary region in front of them has the same alignment.
__device__ __forceinline__ uint8_t *pool_end(uint8_t *pool, int32_t p) { return pool + ((int64_t)p + 1) * kCarryWindow; }

__global__ void __launch_bounds__(kCarryThreads)
    k_carry_stage(const CarrySlot *__restrict__ slots, uint8_t *__restrict__ pool, const uint8_t *__restrict__ packed, uint8_t *__restrict__ in) {
	const CarrySlot s = slots[blockIdx.x];
	cta_copy(in + s.data_off - s.win_len, pool_end(pool, s.pool) - s.win_len, s.win_len);
	cta_copy(in + s.data_off, packed + s.pk_off, s.comp);
}

// the last min(32768, win_len + out_pos) bytes of (old window ++ the run's first out_pos output bytes); the old window is
// read from the slot the run decoded from, so the pool slot written is never read
__global__ void __launch_bounds__(kCarryThreads)
    k_carry_window(const CarrySlot *__restrict__ slots, const uint8_t *__restrict__ in, const uint8_t *__restrict__ out, uint8_t *__restrict__ pool) {
	const CarrySlot s = slots[blockIdx.x];
	const int64_t m = s.out_pos < kCarryWindow ? s.out_pos : kCarryWindow;
	const int64_t keep = s.win_len < kCarryWindow - m ? s.win_len : kCarryWindow - m;
	uint8_t *end = pool_end(pool, s.pool);
	cta_copy(end - m - keep, in + s.data_off - keep, keep);
	cta_copy(end - m, out + s.out_off + s.out_pos - m, m);
}

int carry_stage_launch(const CarrySlot *d_slots, int32_t k, uint8_t *d_pool, const uint8_t *d_packed, uint8_t *d_in, cudaStream_t s) {
	if (k > 0) k_carry_stage<<<k, kCarryThreads, 0, s>>>(d_slots, d_pool, d_packed, d_in);
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

int carry_window_launch(const CarrySlot *d_slots, int32_t k, const uint8_t *d_in, const uint8_t *d_out, uint8_t *d_pool, cudaStream_t s) {
	if (k > 0) k_carry_window<<<k, kCarryThreads, 0, s>>>(d_slots, d_in, d_out, d_pool);
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

} // namespace b200z
