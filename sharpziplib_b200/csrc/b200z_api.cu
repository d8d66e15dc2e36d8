// b200z_api.cu -- the C-ABI of libb200z.so (include/b200z.h): context and errors, the static tables, plans and the
// checksum entry points.  The host-buffer pipelines and batch calls are in b200z_host.cu, the streaming handles in
// b200z_handles.cu.  No CPU codec lives here: every byte of compressed or decompressed data is produced by the kernels in
// b200z_deflate.cu / b200z_inflate.cu.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "b200z_internal.cuh"
#include <dlfcn.h>

namespace b200z {

static thread_local std::string g_err;
static std::mutex g_mu;
thread_local int t_device = -1;

void set_error(const char *fmt, ...) {
	char buf[512];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof(buf), fmt, ap);
	va_end(ap);
	g_err = buf;
}

int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
	set_error("CUDA error %d (%s) at %s:%d in %s", (int)e, cudaGetErrorString(e), file, line, what);
	return B200Z_E_CUDA;
}

int ensure_init() {
	std::lock_guard<std::mutex> lk(g_mu);
	if (t_device >= 0) return B200Z_OK;
	int cnt = 0;
	cudaError_t e = cudaGetDeviceCount(&cnt);
	if (e != cudaSuccess || cnt == 0) {
		set_error("no CUDA device: libb200z has no CPU fallback (%s)", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
		return B200Z_E_CUDA;
	}
	int dev = 0;
	B200Z_CUDA(cudaGetDevice(&dev));
	t_device = dev;
	return B200Z_OK;
}

int current_device() {
	if (t_device >= 0) return t_device;
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) return -1;
	return dev;
}

int Arena::alloc() {
	size = align_up(used + 256, 256);
	cudaError_t e = cudaMalloc(&base, (size_t)size);
	if (e != cudaSuccess) {
		base = nullptr;
		set_error("cudaMalloc of %lld workspace bytes failed: %s", (long long)size, cudaGetErrorString(e));
		return B200Z_E_NOMEM;
	}
	for (const auto &u : pending)
		if (!u.second.empty()) B200Z_CUDA(cudaMemcpy(base + u.first, u.second.data(), u.second.size(), cudaMemcpyHostToDevice));
	pending.clear();
	return B200Z_OK;
}

// ---- static tables blob ---------------------------------------------------------------------------
static void fill_static_blob(uint8_t *b) {
	// encoder side: DeflaterHuffman static ctor (:602-642); decoder side: InflaterHuffmanTree static ctor (:34-70)
	size_t o = 0;
	for (int i = 0; i < kLiteralNum; i++) {
		uint16_t c = (uint16_t)static_lcode(i);
		memcpy(b + o, &c, 2);
		o += 2;
	}
	for (int i = 0; i < kLiteralNum; i++) b[o++] = (uint8_t)static_llen(i);
	for (int i = 0; i < kDistNum; i++) {
		uint16_t c = (uint16_t)static_dcode(i);
		memcpy(b + o, &c, 2);
		o += 2;
	}
	for (int i = 0; i < kDistNum; i++) b[o++] = 5;
	for (int i = 0; i < 288; i++) b[o++] = (uint8_t)(i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8)));
	for (int i = 0; i < 32; i++) b[o++] = 5;
}
constexpr int kStaticBlob = kLiteralNum * 3 + kDistNum * 3 + 288 + 32;

// ---- packing the produced streams back to back (so a caller copies only what was produced) -----------------
__global__ void k_pack_offsets(int n, const int64_t *__restrict__ len, int64_t *__restrict__ off) {
	// n is a batch size (thousands at most): one thread block, serial carry between 1024-element chunks
	__shared__ int64_t s_part[32];
	__shared__ int64_t s_carry;
	if (threadIdx.x == 0) s_carry = 0;
	__syncthreads();
	for (int base = 0; base < n; base += 1024) {
		const int i = base + threadIdx.x;
		const int64_t v = i < n ? ((len[i] + 15) & ~15ll) : 0; // 16-byte aligned starts: vector copies on both sides
		int64_t incl = v;
		for (int o = 1; o < 32; o <<= 1) {
			const int64_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if ((threadIdx.x & 31) >= o) incl += t;
		}
		if ((threadIdx.x & 31) == 31) s_part[threadIdx.x >> 5] = incl;
		__syncthreads();
		int64_t woff = 0;
		for (int k = 0; k < (int)(threadIdx.x >> 5); k++) woff += s_part[k];
		const int64_t carry = s_carry;
		if (i < n) off[i] = carry + woff + incl - v;
		__syncthreads();
		if (threadIdx.x == 1023) s_carry = carry + woff + incl;
		__syncthreads();
	}
	if (threadIdx.x == 0) off[n] = s_carry;
}

__global__ void __launch_bounds__(256)
    k_pack(const uint8_t *__restrict__ out, const int64_t *__restrict__ out_off, const int64_t *__restrict__ len,
           const int64_t *__restrict__ off, uint8_t *__restrict__ packed) {
	const int i = blockIdx.x;
	const uint8_t *src = out + out_off[i];
	uint8_t *dst = packed + off[i];
	const int64_t nb = len[i];
	const int64_t nv = (nb + 15) >> 4; // the slot is 256-byte aligned and at least 16 bytes longer than the data
	const uint4 *sv = reinterpret_cast<const uint4 *>(src);
	uint4 *dv = reinterpret_cast<uint4 *>(dst);
	for (int64_t k = threadIdx.x; k < nv; k += blockDim.x) dv[k] = sv[k];
}

static int checksum_host(int kind, const uint8_t *buf, int64_t len, uint32_t *value) {
	if (!value || len < 0 || (len > 0 && !buf)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	if (len == 0) return B200Z_OK;
	DevBuf d, meta;
	if ((rc = d.ensure((size_t)len + 256))) return rc;
	B200Z_CUDA(cudaMemcpy(d.p, buf, (size_t)len, cudaMemcpyHostToDevice));
	std::vector<CkTile> tiles;
	checksum_tiles(&len, 1, tiles, kind);
	const size_t tb = sizeof(CkTile) * tiles.size();
	if ((rc = meta.ensure(tb + 256))) return rc;
	int64_t *d_off = reinterpret_cast<int64_t *>(meta.p);
	int64_t *d_len = d_off + 1;
	unsigned long long *d_acc = reinterpret_cast<unsigned long long *>(d_len + 1);
	uint32_t *d_val = reinterpret_cast<uint32_t *>(d_acc + 2);
	CkTile *d_tiles = reinterpret_cast<CkTile *>(meta.p + 64);
	int64_t zero = 0;
	B200Z_CUDA(cudaMemcpy(d_off, &zero, 8, cudaMemcpyHostToDevice));
	B200Z_CUDA(cudaMemcpy(d_len, &len, 8, cudaMemcpyHostToDevice));
	B200Z_CUDA(cudaMemcpy(d_val, value, 4, cudaMemcpyHostToDevice));
	B200Z_CUDA(cudaMemcpy(d_tiles, tiles.data(), tb, cudaMemcpyHostToDevice));
	rc = checksum_launch(kind, d.p, d_off, d_len, 1, d_tiles, (int32_t)tiles.size(), d_acc, d_val, 0, 0, false);
	if (rc) return rc;
	B200Z_CUDA(cudaMemcpy(value, d_val, 4, cudaMemcpyDeviceToHost));
	return B200Z_OK;
}

} // namespace b200z

using namespace b200z;

extern "C" {

const char *b200z_last_error(void) { return g_err.c_str(); }
int b200z_version(void) { return 100; }

int b200z_init(int device) {
	{
		std::lock_guard<std::mutex> lk(g_mu);
		int cnt = 0;
		cudaError_t e = cudaGetDeviceCount(&cnt);
		if (e != cudaSuccess || cnt == 0) {
			set_error("no CUDA device: libb200z has no CPU fallback (%s)", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
			return B200Z_E_CUDA;
		}
		if (device < 0 || device >= cnt) {
			set_error("device %d out of range (%d devices)", device, cnt);
			return B200Z_E_ARG;
		}
		B200Z_CUDA(cudaSetDevice(device));
		t_device = device;
	}
	return checksum_init_tables();
}

int b200z_static_tables_size(void) { return kStaticBlob; }
int b200z_static_tables_export(uint8_t *blob, int32_t cap) {
	if (!blob || cap < kStaticBlob) {
		set_error("static table blob needs %d bytes", kStaticBlob);
		return B200Z_E_ARG;
	}
	fill_static_blob(blob);
	return B200Z_OK;
}
int b200z_static_tables_import(const uint8_t *blob, int32_t len) {
	// The kernels derive the static codes arithmetically (b200z_core.cuh static_lcode/static_llen), so installing a
	// broadcast copy reduces to verifying that the sender's tables are the ones this rank would use.
	if (!blob || len != kStaticBlob) {
		set_error("static table blob has %d bytes, expected %d", len, kStaticBlob);
		return B200Z_E_ARG;
	}
	uint8_t mine[kStaticBlob];
	fill_static_blob(mine);
	if (memcmp(mine, blob, kStaticBlob) != 0) {
		set_error("static Huffman tables received from the root differ from the local ones");
		return B200Z_E_DATA;
	}
	return B200Z_OK;
}

// ncclBroadcast inside the library, for a host that owns a communicator (one process per GPU).  NCCL is not linked: the
// two entry points are taken from the libnccl the process has loaded (or can load) at run time.
typedef int (*nccl_bcast_fn)(const void *, void *, size_t, int, int, void *, cudaStream_t);
typedef const char *(*nccl_errstr_fn)(int);
int b200z_static_tables_broadcast(void *nccl_comm, int32_t root, int32_t rank, void *cuda_stream) {
	if (!nccl_comm || root < 0 || rank < 0) {
		set_error("b200z_static_tables_broadcast: communicator, root and rank are required");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	static nccl_bcast_fn bcast = nullptr;
	static nccl_errstr_fn errstr = nullptr;
	if (!bcast) {
		void *h = nullptr;
		const char *names[] = {"libnccl.so.2", "libnccl.so"};
		for (int k = 0; k < 2 && !h; k++) h = dlopen(names[k], RTLD_NOW | RTLD_NOLOAD);
		for (int k = 0; k < 2 && !h; k++) h = dlopen(names[k], RTLD_NOW | RTLD_GLOBAL);
		if (h) {
			bcast = (nccl_bcast_fn)dlsym(h, "ncclBroadcast");
			errstr = (nccl_errstr_fn)dlsym(h, "ncclGetErrorString");
		}
		if (!bcast) {
			set_error("b200z_static_tables_broadcast: no libnccl in this process (dlopen libnccl.so.2 failed)");
			return B200Z_E_UNSUPPORTED;
		}
	}
	cudaStream_t s = (cudaStream_t)cuda_stream;
	DevBuf d;
	if ((rc = d.ensure(kStaticBlob))) return rc;
	uint8_t blob[kStaticBlob];
	if (rank == root) {
		fill_static_blob(blob);
		B200Z_CUDA(cudaMemcpyAsync(d.p, blob, kStaticBlob, cudaMemcpyHostToDevice, s));
	}
	const int nr = bcast(d.p, d.p, (size_t)kStaticBlob, /* ncclUint8 */ 1, root, nccl_comm, s);
	if (nr != 0) {
		set_error("ncclBroadcast failed: %s", errstr ? errstr(nr) : "?");
		return B200Z_E_CUDA;
	}
	B200Z_CUDA(cudaMemcpyAsync(blob, d.p, kStaticBlob, cudaMemcpyDeviceToHost, s));
	B200Z_CUDA(cudaStreamSynchronize(s));
	return b200z_static_tables_import(blob, kStaticBlob);
}

int64_t b200z_deflate_bound(int64_t len) { return len + (len >> 3) + 1024; }
int64_t b200z_engine_state_bytes(void) { return kFastStateBytes; }

// ---- plans -------------------------------------------------------------------------------------------
int b200z_deflate_plan_create(int32_t n, const int64_t *in_len, int level, int strategy, int wrap, int end_mode,
                              b200z_plan **plan) {
	return b200z_deflate_plan_create_ex(n, in_len, level, strategy, wrap, end_mode, nullptr, plan);
}

int b200z_deflate_plan_create_ex(int32_t n, const int64_t *in_len, int level, int strategy, int wrap, int end_mode,
                                 const b200z_history *hist, b200z_plan **plan) {
	if (!plan || n < 0 || (n > 0 && !in_len)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (level == -1) level = 6;
	if (level < 0 || level > 9) {
		set_error("level");
		return B200Z_E_ARG;
	}
	if (strategy < 0 || strategy > 2 || wrap < 0 || wrap > B200Z_WRAP_RAW_CRC32 || end_mode < 0 || end_mode > B200Z_END_NONE) {
		set_error("strategy/wrap/end_mode");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	DeviceGuard guard(current_device());
	return deflate_plan_create(n, in_len, level, strategy, wrap, end_mode, hist, plan);
}

int b200z_deflate_plan_set_entry(b200z_plan *plan, const b200z_parse_entry *entry) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 0 || (plan->n > 0 && !entry)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	return deflate_plan_set_entry(plan, entry);
}

int b200z_deflate_plan_get_cut(b200z_plan *plan, int64_t *covered, b200z_parse_entry *next, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 0 || (plan->n > 0 && (!covered || (!next && plan->level >= 5)))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	return deflate_plan_get_cut(plan, covered, next, (cudaStream_t)cuda_stream);
}

int b200z_deflate_plan_get_cut_call(b200z_plan *plan, int32_t *call, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 0 || (plan->n > 0 && !call)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	return deflate_plan_get_cut_call(plan, call, (cudaStream_t)cuda_stream);
}

int b200z_inflate_plan_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, int wrap, b200z_plan **plan) {
	return b200z_inflate_plan_create_ex(n, comp_len, out_cap, wrap, nullptr, plan);
}

int b200z_inflate_plan_create_ex(int32_t n, const int64_t *comp_len, const int64_t *out_cap, int wrap, const int64_t *dict_len,
                                 b200z_plan **plan) {
	if (!plan || n < 0 || (n > 0 && (!comp_len || !out_cap)) || wrap < 0 || wrap > B200Z_WRAP_RAW_CRC32) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	DeviceGuard guard(current_device());
	return inflate_plan_create(n, comp_len, out_cap, wrap, dict_len, plan);
}

int b200z_lzw_plan_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, b200z_plan **plan) {
	if (!plan || n < 0 || (n > 0 && (!comp_len || !out_cap))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	DeviceGuard guard(current_device());
	return lzw_plan_create(n, comp_len, out_cap, plan);
}

int b200z_inflate_plan_set_start_bits(b200z_plan *plan, const int32_t *start_bit) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 1 || (plan->n > 0 && !start_bit)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->wrap != B200Z_WRAP_RAW && plan->wrap != B200Z_WRAP_RAW_CRC32) {
		set_error("start bits are for raw streams (a framed stream starts behind its header)");
		return B200Z_E_ARG;
	}
	for (int i = 0; i < plan->n; i++) {
		if (start_bit[i] < 0 || start_bit[i] > 7) {
			set_error("stream %d: start bit %d (0..7)", i, start_bit[i]);
			return B200Z_E_ARG;
		}
	}
	return inflate_plan_set_start_bits(plan, start_bit);
}

int b200z_inflate_plan_set_resume(b200z_plan *plan, const int32_t *start_bit, const int64_t *skip_bit) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 1 || (plan->n > 0 && (!start_bit || !skip_bit))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->wrap != B200Z_WRAP_RAW) {
		set_error("resume points are for raw streams");
		return B200Z_E_ARG;
	}
	for (int i = 0; i < plan->n; i++) {
		if (start_bit[i] < 0 || start_bit[i] > 7 || skip_bit[i] < 0 || skip_bit[i] > 0x7FFFFFFF8ll) {
			set_error("stream %d: start bit %d (0..7), skip bit %lld", i, start_bit[i], (long long)skip_bit[i]);
			return B200Z_E_ARG;
		}
	}
	return inflate_plan_set_resume(plan, start_bit, skip_bit);
}

int b200z_inflate_plan_set_lengths(b200z_plan *plan, const int64_t *comp_len, const int64_t *dict_len) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 1 || (plan->n > 0 && !comp_len)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	return inflate_plan_set_lengths(plan, comp_len, dict_len);
}

int b200z_plan_get_restart_points(b200z_plan *plan, int64_t *bit, int64_t *out_pos, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 1 || (plan->n > 0 && (!bit || !out_pos))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->n == 0) return B200Z_OK;
	return inflate_plan_restart_points(plan, bit, out_pos, (cudaStream_t)cuda_stream);
}

int b200z_plan_get_resume_points(b200z_plan *plan, int64_t *hdr_bit, int64_t *body_bit, int64_t *sym_bit, int64_t *out_pos,
                                 void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind != 1 || (plan->n > 0 && (!hdr_bit || !body_bit || !sym_bit || !out_pos))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->n == 0) return B200Z_OK;
	return inflate_plan_resume_points(plan, hdr_bit, body_bit, sym_bit, out_pos, (cudaStream_t)cuda_stream);
}

int b200z_plan_get_stats(b200z_plan *plan, uint32_t *v, int32_t cap, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || plan->kind == 0 || !v || cap < 0) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->kind == 2) return lzw_plan_stats(plan, v, cap, (cudaStream_t)cuda_stream);
	return inflate_plan_stats(plan, v, cap, (cudaStream_t)cuda_stream);
}

int b200z_plan_set_timing(b200z_plan *plan, int enable) {
	if (!plan) return B200Z_E_ARG;
	plan->timing = enable != 0;
	plan->ev_used = 0;
	return B200Z_OK;
}

int b200z_plan_get_timings(b200z_plan *plan, char *names, int32_t names_cap, float *ms, int32_t cap, int32_t *count) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || !ms || !count) return B200Z_E_ARG;
	*count = 0;
	std::string nm;
	for (int i = 0; i + 1 < plan->ev_used && *count < cap; i++) {
		float t = 0;
		cudaError_t e = cudaEventElapsedTime(&t, plan->ev[i], plan->ev[i + 1]);
		if (e != cudaSuccess) return cuda_fail(e, "cudaEventElapsedTime", __FILE__, __LINE__);
		ms[*count] = t;
		nm += plan->ev_name[i];
		nm += ";";
		++*count;
	}
	if (names && names_cap > 0) {
		strncpy(names, nm.c_str(), (size_t)names_cap - 1);
		names[names_cap - 1] = 0;
	}
	return B200Z_OK;
}

int b200z_plan_destroy(b200z_plan *plan) {
	DeviceGuard guard(plan ? plan->device : -1);
	delete plan;
	return B200Z_OK;
}
int64_t b200z_plan_in_bytes(const b200z_plan *p) { return p->in_bytes; }
int64_t b200z_plan_out_bytes(const b200z_plan *p) { return p->out_bytes; }
int64_t b200z_plan_in_offset(const b200z_plan *p, int32_t i) { return p->in_off[i]; }
int64_t b200z_plan_data_offset(const b200z_plan *p, int32_t i) {
	return p->in_off[i] + (p->hist.empty() ? 0 : p->hist[i]); // behind the history / dictionary
}
int64_t b200z_plan_out_offset(const b200z_plan *p, int32_t i) { return p->out_off[i]; }
int64_t b200z_plan_out_capacity(const b200z_plan *p, int32_t i) { return p->out_cap[i]; }
int64_t b200z_plan_workspace_bytes(const b200z_plan *p) { return p->ws.size; }
int32_t b200z_plan_launches(const b200z_plan *p) { return p->launches; }

int b200z_plan_run(b200z_plan *plan, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                   uint32_t *d_check, int64_t *d_in_used, void *cuda_stream) {
	return b200z_plan_run_stages(plan, d_in, d_out, d_out_len, d_status, d_check, d_in_used, B200Z_STAGE_SEARCH | B200Z_STAGE_ENCODE,
	                             cuda_stream);
}

int b200z_plan_run_stages(b200z_plan *plan, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                          uint32_t *d_check, int64_t *d_in_used, int stages, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || !d_in || !d_out || !d_out_len || !d_status || (stages & ~3) || stages == 0) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	cudaStream_t s = (cudaStream_t)cuda_stream;
	if (plan->kind == 0) return deflate_plan_run(plan, d_in, d_out, d_out_len, d_status, d_check, d_in_used, s, stages);
	if (!(stages & B200Z_STAGE_ENCODE)) return B200Z_OK; // inflate and LZW plans are a single stage
	if (plan->kind == 2) return lzw_plan_run(plan, d_in, d_out, d_out_len, d_status, d_check, d_in_used, s);
	return inflate_plan_run(plan, d_in, d_out, d_out_len, d_status, d_check, d_in_used, s);
}

int b200z_plan_pack(b200z_plan *plan, const uint8_t *d_out, const int64_t *d_out_len, uint8_t *d_packed,
                    int64_t *d_packed_off, void *cuda_stream) {
	DeviceGuard guard(plan ? plan->device : -1);
	if (!plan || !d_out || !d_out_len || !d_packed || !d_packed_off) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (plan->kind == 2) { // a stream that did not fit reports the size it needs in d_out_len, not bytes in d_out
		set_error("LZW plans are not packed: a B200Z_E_NOMEM stream's out_len is the size it needs, not bytes of its slot");
		return B200Z_E_UNSUPPORTED;
	}
	if (plan->n == 0) return B200Z_OK;
	cudaStream_t s = (cudaStream_t)cuda_stream;
	k_pack_offsets<<<1, 1024, 0, s>>>(plan->n, d_out_len, d_packed_off);
	k_pack<<<plan->n, 256, 0, s>>>(d_out, plan->dev_out_off(), d_out_len, d_packed_off, d_packed);
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

// ---- checksums ---------------------------------------------------------------------------------------
int b200z_crc32(const uint8_t *buf, int64_t len, uint32_t *value) { return checksum_host(0, buf, len, value); }
int b200z_bzip2crc(const uint8_t *buf, int64_t len, uint32_t *value) { return checksum_host(2, buf, len, value); }
int b200z_adler32(const uint8_t *buf, int64_t len, uint32_t *value) { return checksum_host(1, buf, len, value); }

int b200z_checksum_batch_device(int kind, const uint8_t *d_data, const int64_t *off, const int64_t *len, int32_t n,
                                uint32_t *d_value, void *cuda_stream) {
	if (kind < 0 || kind > 2 || n < 0 || (n > 0 && (!d_data || !off || !len || !d_value))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	if (n == 0) return B200Z_OK;
	cudaStream_t s = (cudaStream_t)cuda_stream;
	std::vector<CkTile> tiles;
	checksum_tiles(len, n, tiles, kind);
	const size_t tb = sizeof(CkTile) * tiles.size();
	uint8_t *meta = nullptr;
	const size_t bytes = 16ull * n + 16ull * n + tb + 256;
	B200Z_CUDA(cudaMallocAsync((void **)&meta, bytes, s));
	int64_t *d_off = reinterpret_cast<int64_t *>(meta);
	int64_t *d_len = d_off + n;
	unsigned long long *d_acc = reinterpret_cast<unsigned long long *>(d_len + n);
	CkTile *d_tiles = reinterpret_cast<CkTile *>(d_acc + 2 * n);
	B200Z_CUDA(cudaMemcpyAsync(d_off, off, 8ull * n, cudaMemcpyHostToDevice, s));
	B200Z_CUDA(cudaMemcpyAsync(d_len, len, 8ull * n, cudaMemcpyHostToDevice, s));
	if (tb) B200Z_CUDA(cudaMemcpyAsync(d_tiles, tiles.data(), tb, cudaMemcpyHostToDevice, s));
	rc = checksum_launch(kind, d_data, d_off, d_len, n, d_tiles, (int32_t)tiles.size(), d_acc, d_value, 0, s, false);
	B200Z_CUDA(cudaStreamSynchronize(s)); // the pageable descriptor copies above must finish before `tiles` dies
	B200Z_CUDA(cudaFreeAsync(meta, s));
	return rc;
}

} // extern "C"
