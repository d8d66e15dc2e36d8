// b200z_host.cuh -- what the host-buffer pipelines (b200z_host.cu) and the streaming handles (b200z_handles.cu) share:
// the staging of one plan run between host buffers and the device, and the zlib framing helpers.
#pragma once
#include "b200z_internal.cuh"

namespace b200z {

struct PipeMeta { // what a run reports, per stream; poff (n + 1 entries) is written only by a pack
	int64_t *out_len, *in_used;
	int32_t *status;
	uint32_t *check;
	int64_t *poff;
};

// A plan's input and output blobs in pinned and device memory, and its metadata on both sides (h, d).  dpack, the
// produced streams packed back to back, exists only when ensure() is asked for it.
struct Staging {
	PinnedBuf hin, hout;
	DevBuf din, dout, dpack;
	PipeMeta h, d;
	int ensure(const b200z_plan *plan, bool pack); // grows every buffer to the plan's blobs
};

// Enqueues a run: on `up` the inputs (the DMA source is in[i] itself when the caller knows them as pinned, hin otherwise,
// and then only the used prefix of the blob) and the optional running checksum seed; on `run`, behind ev_up when one is
// given, the plan's kernels, the pack when dpack exists and the metadata down into h.
int stage_run(b200z_plan *plan, Staging &st, const uint8_t *const *in, bool in_pinned, const uint32_t *check_seed, cudaStream_t up,
              cudaStream_t run, cudaEvent_t ev_up);
// Once h holds the run's lengths: the produced bytes of every stream down into dst[i], or into hout at the stream's
// out_off when dst is null, on `s`; returns when they are there.
int streams_down(const b200z_plan *plan, Staging &st, uint8_t *const *dst, cudaStream_t s);

void zlib_header(int level, uint8_t h[2], bool preset_dict = false);
const char *inflate_detail_msg(int detail); // the reference's exception message for an inflate status detail
std::string lzw_detail_msg(int32_t status, uint32_t value); // the reference's message for an LZW status and its numbers

} // namespace b200z
