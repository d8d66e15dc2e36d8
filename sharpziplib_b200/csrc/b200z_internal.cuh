// b200z_internal.cuh -- shared host-side plumbing of libb200z.so (context, error reporting, plan object).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200z.h"
#include "b200z_core.cuh"
#include "b200z_crc.cuh"

namespace b200z {

void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define B200Z_CUDA(call)                                                                   \
	do {                                                                                   \
		cudaError_t e__ = (call);                                                          \
		if (e__ != cudaSuccess) return ::b200z::cuda_fail(e__, #call, __FILE__, __LINE__); \
	} while (0)

int ensure_init(); // picks up the current device if b200z_init() was not called explicitly
int current_device(); // the device b200z_init() chose for the calling thread (the CUDA current device otherwise)
extern thread_local int t_device; // what b200z_init() chose for the calling thread, -1 before

// Every object (plan, pipeline, handle) remembers the device it was created on; its entry points run there and leave the
// calling thread's current device as they found it, so that one host thread can drive several GPUs.
struct DeviceGuard {
	int prev = -1;
	explicit DeviceGuard(int dev) {
		if (dev < 0) return;
		int cur = -1;
		if (cudaGetDevice(&cur) == cudaSuccess && cur != dev) {
			prev = cur;
			cudaSetDevice(dev);
		}
	}
	~DeviceGuard() {
		if (prev >= 0) cudaSetDevice(prev);
	}
};

constexpr int64_t kAlign = 256; // stream slots in the blobs start on 256-byte boundaries (vector loads / bulk copies)
inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

template <class T> struct Slot;

// An owned allocation of pinned host (Pinned) or device memory.  ensure() grows it and does not keep the contents.
template <bool Pinned> struct Buf {
	uint8_t *p = nullptr;
	size_t cap = 0;
	Buf() = default;
	Buf(Buf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; } // (not copyable)
	~Buf() { release(); }
	int ensure(size_t n) {
		if (n <= cap) return B200Z_OK;
		release();
		const cudaError_t e = Pinned ? cudaHostAlloc((void **)&p, n, cudaHostAllocDefault) : cudaMalloc((void **)&p, n);
		if (e != cudaSuccess) {
			p = nullptr;
			set_error("%s of %zu bytes failed: %s", Pinned ? "cudaHostAlloc" : "cudaMalloc", n, cudaGetErrorString(e));
			return B200Z_E_NOMEM;
		}
		cap = n;
		return B200Z_OK;
	}
	void release() {
		if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
		p = nullptr;
		cap = 0;
	}
	template <class T> T *at(Slot<T> s) const { return reinterpret_cast<T *>(p + s.off); } // a slot an Arena laid out
};
using PinnedBuf = Buf<true>;
using DevBuf = Buf<false>;

// The SM count of the calling thread's current device.
inline cudaError_t sm_count(int *sms) {
	int dev = 0;
	const cudaError_t e = cudaGetDevice(&dev);
	return e == cudaSuccess ? cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev) : e;
}

// An array of T in an Arena.
template <class T> struct Slot {
	int64_t off = 0;
};

// One device allocation carved into typed arrays: a plan reserves and uploads its arrays, then alloc() allocates them all
// and copies in what upload() was given.
struct Arena {
	uint8_t *base = nullptr;
	int64_t size = 0, used = 0;
	std::vector<std::pair<int64_t, std::vector<uint8_t>>> pending; // (offset, host bytes) that alloc() copies
	template <class T> Slot<T> reserve(int64_t count) {
		const int64_t off = align_up(used, 256);
		used = off + (int64_t)sizeof(T) * count;
		return Slot<T>{off};
	}
	// reserves v.size() + spare elements; alloc() fills the first v.size() of them with v
	template <class T> Slot<T> upload(const std::vector<T> &v, int64_t spare = 0) {
		const Slot<T> s = reserve<T>((int64_t)v.size() + spare);
		const uint8_t *b = reinterpret_cast<const uint8_t *>(v.data());
		pending.emplace_back(s.off, std::vector<uint8_t>(b, b + sizeof(T) * v.size()));
		return s;
	}
	// after alloc(): copies v over the start of the slot
	template <class T> int write(Slot<T> s, const std::vector<T> &v) {
		if (!v.empty()) B200Z_CUDA(cudaMemcpy(at(s), v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
		return B200Z_OK;
	}
	int alloc(); // the plan that owns the arena frees base
	template <class T> T *at(Slot<T> s) const { return reinterpret_cast<T *>(base + s.off); }
};

// per-block tables produced by k_plan and consumed by k_emit
struct __align__(16) BlockTables {
	uint16_t lit_codes[kLiteralNum];
	uint16_t dist_codes[kDistNum];
	uint8_t lit_len[kLiteralNum];
	uint8_t dist_len[kDistNum];
	uint32_t hdr[kHdrWords];
};

struct __align__(16) BlockMeta {
	uint32_t byte_start; // first input byte covered by the block
	uint32_t byte_len;   // storedLength
	uint32_t nsyms;
	uint32_t hdr_bits;
	uint32_t body_bits;
	uint32_t type; // 0 stored, 1 static, 2 dynamic
	uint64_t bit_off; // absolute bit offset inside the stream's output slot (k_scan)
};

// Inflate: one LZ77 back-reference to resolve (phase 2)
struct __align__(8) MatchTok {
	uint32_t out_pos;
	uint16_t len;
	uint16_t dist;
};

} // namespace b200z

// What the C-ABI and the host pipelines see of a plan.  Each pipeline derives its plan type from this one, next to its
// kernels (DeflatePlan in b200z_deflate.cu, InflatePlan in b200z_inflate.cu), and lays out the rest of its workspace there.
struct b200z_plan {
	virtual ~b200z_plan() {
		for (cudaEvent_t e : ev) cudaEventDestroy(e);
		if (ws.base) cudaFree(ws.base);
	}
	int kind = 0; // 0 deflate, 1 inflate, 2 LZW
	int device = -1; // the device the plan's workspace lives on
	int n = 0;
	int level = 6, strategy = 0, wrap = 0, end_mode = 0;
	std::vector<int64_t> in_len, in_off, out_off, out_cap;
	int64_t in_bytes = 0, out_bytes = 0;
	// deflate with history (b200z_deflate_plan_create_ex): in_len[] is history + data; an inflate plan keeps the
	// preset-dictionary lengths in hist[]
	std::vector<int64_t> hist;
	b200z::Arena ws;
	// per stream on the device: where the kernels find its input and how long it is, where its output goes and how much
	// room it has (upload_streams)
	b200z::Slot<int64_t> o_in_off, o_in_len, o_out_off, o_out_cap;
	int launches = 0;
	// reserves the four per-stream tables, each with `spare` unused entries behind the n, and queues their upload
	void upload_streams(const std::vector<int64_t> &dev_in_off, const std::vector<int64_t> &dev_in_len, int spare) {
		o_in_off = ws.upload(dev_in_off, spare);
		o_in_len = ws.upload(dev_in_len, spare);
		o_out_off = ws.upload(out_off, spare);
		o_out_cap = ws.upload(out_cap, spare);
	}
	const int64_t *dev_out_off() const { return ws.at(o_out_off); }
	// optional per-kernel timing (b200z_plan_set_timing): events recorded on the run's stream between kernels
	bool timing = false;
	std::vector<cudaEvent_t> ev;
	std::vector<const char *> ev_name; // ev_name[i] labels the interval ev[i] -> ev[i+1]
	int ev_used = 0;
	void mark(cudaStream_t s, const char *next_name) {
		if (!timing) return;
		if ((int)ev.size() <= ev_used) {
			cudaEvent_t e;
			cudaEventCreate(&e);
			ev.push_back(e);
			ev_name.push_back("");
		}
		cudaEventRecord(ev[ev_used], s);
		ev_name[ev_used] = next_name;
		++ev_used;
	}
};

namespace b200z {
// implemented in b200z_deflate.cu / b200z_inflate.cu / b200z_checksum.cu; the create functions take arguments the C-ABI
// has checked and validate the history / dictionary lengths themselves
int deflate_plan_create(int32_t n, const int64_t *in_len, int level, int strategy, int wrap, int end_mode,
                        const b200z_history *hist, b200z_plan **out);
int deflate_plan_run(b200z_plan *p, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                     uint32_t *d_check, int64_t *d_out_bits, cudaStream_t s, int stages);
int deflate_plan_set_entry(b200z_plan *p, const b200z_parse_entry *entry);
int deflate_plan_get_cut(b200z_plan *p, int64_t *covered, b200z_parse_entry *next, cudaStream_t s);
int deflate_plan_get_cut_call(b200z_plan *p, int32_t *call, cudaStream_t s);
int inflate_plan_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, int wrap, const int64_t *dict_len,
                        b200z_plan **out);
int inflate_plan_set_start_bits(b200z_plan *p, const int32_t *start_bit);
int inflate_plan_set_lengths(b200z_plan *p, const int64_t *comp_len, const int64_t *dict_len);
int inflate_plan_restart_points(b200z_plan *p, int64_t *bit, int64_t *out_pos, cudaStream_t s);
int inflate_plan_set_resume(b200z_plan *p, const int32_t *start_bit, const int64_t *skip_bit);
int inflate_plan_resume_points(b200z_plan *p, int64_t *hdr_bit, int64_t *body_bit, int64_t *sym_bit, int64_t *out_pos,
                               cudaStream_t s);
int inflate_plan_stats(b200z_plan *p, uint32_t *v, int32_t cap, cudaStream_t s);
int inflate_plan_run(b200z_plan *p, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                     uint32_t *d_check, int64_t *d_in_used, cudaStream_t s);
// checksum over n device buffers (kind 0 = CRC32, 1 = Adler32, 2 = CRC-32/BZIP2); d_acc = 2 x uint64 scratch per stream;
// value in/out (device uint32), `fresh` != 0 starts from the Reset() value instead of reading d_value.
// `dynamic`: the tiles were laid over capacities (checksum_tiles(..., dynamic = true)) and d_len holds the real lengths,
// known only on the device: the kernel skips the tiles past them and works the multipliers out itself (kinds 0 and 1 only).
int checksum_launch(int kind, const uint8_t *d_data, const int64_t *d_off, const int64_t *d_len, int32_t n,
                    const CkTile *d_tiles, int32_t n_tiles, unsigned long long *d_acc, uint32_t *d_value, int fresh,
                    cudaStream_t s, bool dynamic);
int checksum_tiles(const int64_t *len, int32_t n, std::vector<CkTile> &tiles, int kind, bool dynamic = false);
int checksum_init_tables();
// b200z_lzw.cu: LZW (.Z) plans; the run reports the numbers of a stream's error message in d_value
int lzw_plan_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, b200z_plan **out);
int lzw_plan_run(b200z_plan *p, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status, uint32_t *d_value,
                 int64_t *d_in_used, cudaStream_t s);
int lzw_plan_stats(b200z_plan *p, uint32_t *v, int32_t cap, cudaStream_t s);
// b200z_inflate_streams.cu: the window pool of the inflate carry.  Pool slot p is kCarryWindow bytes; its window is the
// slot's last win_len bytes.  Per stream of a run: the packed upload holds comp bytes (header copy, then compressed bytes)
// at pk_off; the plan's compressed bytes start at data_off of the input blob, the window in front of them; out_pos is the
// output the window moves over after the run (k_carry_window).
constexpr int64_t kCarryWindow = 32768;
struct CarrySlot {
	int64_t pk_off, data_off, comp, out_off, out_pos;
	int32_t pool, win_len;
};
int carry_stage_launch(const CarrySlot *d_slots, int32_t k, uint8_t *d_pool, const uint8_t *d_packed, uint8_t *d_in, cudaStream_t s);
int carry_window_launch(const CarrySlot *d_slots, int32_t k, const uint8_t *d_in, const uint8_t *d_out, uint8_t *d_pool, cudaStream_t s);
} // namespace b200z
