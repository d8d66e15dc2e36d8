// b200z_host.cu -- running plans from host buffers: the staging both the pipelines and the streaming handles use, the
// host-buffer pipelines, the batch calls on one device or several, and the byte partition that cuts a batch across devices.
#include <algorithm>
#include <cstring>
#include <functional>
#include <thread>
#include <utility>

#include "b200z_host.cuh"

// ---- host-buffer pipelines ---------------------------------------------------------------------------------
// What a host that keeps a GPU busy does, inside the library: a pipeline owns the plan of one batch shape, `depth` slots of
// pinned staging + device buffers and three streams.  submit() stages a batch from host pointers and enqueues upload and
// kernels without waiting; collect() waits for the oldest batch, fetches exactly the bytes produced and hands them to the
// caller's buffers.  With depth >= 2 the upload of batch i+1 and the download of batch i-1 overlap the kernels of batch i.
// Host pointers that CUDA knows as pinned (cudaHostAlloc / cudaHostRegister) are the DMA source / target directly; plain
// pageable memory goes through the slot's pinned staging, copied by a few host threads.
struct b200z_pipeline {
	struct Slot : b200z::Staging {
		cudaEvent_t ev_up = nullptr, ev_run = nullptr;
	};
	b200z_plan *plan = nullptr;
	int wrap = 0; // the framing collect() writes around the plan's streams
	int depth = 1;
	std::vector<Slot> slots;
	cudaStream_t s_up = nullptr, s_run = nullptr, s_down = nullptr;
	int64_t head = 0, tail = 0; // batches submitted / collected
};

namespace b200z {

static void host_parallel_for(int n_items, int64_t total_bytes, const std::function<void(int, int)> &fn) {
	// fn(first, last) over [0, n_items), on up to 8 threads when there is enough to copy
	int nt = total_bytes >= (8ll << 20) ? std::min(8, n_items) : 1;
	if (nt > 1) { // (hardware_concurrency() is a system call: a handle's run stages one stream and does not ask)
		const int hw = (int)std::thread::hardware_concurrency();
		if (hw > 0 && nt > hw) nt = hw;
	}
	if (nt <= 1) {
		fn(0, n_items);
		return;
	}
	std::vector<std::thread> th;
	for (int t = 0; t < nt; t++) th.emplace_back([=, &fn] { fn((int)((int64_t)n_items * t / nt), (int)((int64_t)n_items * (t + 1) / nt)); });
	for (auto &t : th) t.join();
}

static bool host_ptr_is_pinned(const void *p) {
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
		cudaGetLastError();
		return false;
	}
	return a.type == cudaMemoryTypeHost;
}

// poff last: a run without a pack downloads the first 24 n bytes only
static void pipe_meta_layout(uint8_t *base, int n, PipeMeta &m) {
	m.out_len = reinterpret_cast<int64_t *>(base);
	m.in_used = m.out_len + n;
	m.status = reinterpret_cast<int32_t *>(m.in_used + n);
	m.check = reinterpret_cast<uint32_t *>(m.status + n);
	m.poff = reinterpret_cast<int64_t *>(m.check + n);
}

// The metadata sits behind the output blob in hout and dout: a handle allocates its staging once, and pinned allocations
// are slow.
int Staging::ensure(const b200z_plan *plan, bool pack) {
	const size_t in = (size_t)plan->in_bytes + 256, out = (size_t)plan->out_bytes + 256, meta = (size_t)plan->n * (8 + 8 + 4 + 4 + 8) + 8;
	int rc;
	if ((rc = hin.ensure(in)) || (rc = hout.ensure(out + meta)) || (rc = din.ensure(in)) || (rc = dout.ensure(out + meta)) ||
	    (pack && (rc = dpack.ensure(out))))
		return rc;
	pipe_meta_layout(hout.p + out, plan->n, h);
	pipe_meta_layout(dout.p + out, plan->n, d);
	return B200Z_OK;
}

int stage_run(b200z_plan *plan, Staging &st, const uint8_t *const *in, bool in_pinned, const uint32_t *check_seed, cudaStream_t up,
              cudaStream_t run, cudaEvent_t ev_up) {
	const int n = plan->n;
	if (in_pinned) {
		for (int i = 0; i < n; i++)
			if (plan->in_len[(size_t)i] > 0)
				B200Z_CUDA(cudaMemcpyAsync(st.din.p + plan->in_off[(size_t)i], in[i], (size_t)plan->in_len[(size_t)i], cudaMemcpyHostToDevice, up));
	} else {
		int64_t used = 0, total = 0; // (a plan can run below its capacity: b200z_inflate_plan_set_lengths)
		for (int i = 0; i < n; i++) {
			used = std::max(used, plan->in_off[(size_t)i] + plan->in_len[(size_t)i]);
			total += plan->in_len[(size_t)i];
		}
		host_parallel_for(n, total, [&](int a, int b) {
			for (int i = a; i < b; i++)
				if (plan->in_len[(size_t)i] > 0) memcpy(st.hin.p + plan->in_off[(size_t)i], in[i], (size_t)plan->in_len[(size_t)i]);
		});
		B200Z_CUDA(cudaMemcpyAsync(st.din.p, st.hin.p, (size_t)std::min(plan->in_bytes, align_up(used, 256)), cudaMemcpyHostToDevice, up));
	}
	if (check_seed) B200Z_CUDA(cudaMemcpyAsync(st.d.check, check_seed, 4ull * n, cudaMemcpyHostToDevice, up)); // running values
	if (ev_up) {
		B200Z_CUDA(cudaEventRecord(ev_up, up));
		B200Z_CUDA(cudaStreamWaitEvent(run, ev_up, 0));
	}
	int rc = b200z_plan_run(plan, st.din.p, st.dout.p, st.d.out_len, st.d.status, st.d.check, st.d.in_used, (void *)run);
	if (rc) return rc;
	if (st.dpack.p && (rc = b200z_plan_pack(plan, st.dout.p, st.d.out_len, st.dpack.p, st.d.poff, (void *)run))) return rc;
	const size_t meta = (size_t)n * (8 + 8 + 4 + 4) + (st.dpack.p ? 8ull * (n + 1) : 0);
	B200Z_CUDA(cudaMemcpyAsync(st.h.out_len, st.d.out_len, meta, cudaMemcpyDeviceToHost, run));
	return B200Z_OK;
}

// the bytes a run wrote for stream i: an LZW stream that did not fit reports the size it needs and wrote nothing
static int64_t produced(const b200z_plan *plan, const PipeMeta &m, int i) {
	return plan->kind == 2 && (m.status[i] & 0xFF) == B200Z_E_NOMEM ? 0 : m.out_len[i];
}

int streams_down(const b200z_plan *plan, Staging &st, uint8_t *const *dst, cudaStream_t s) {
	for (int i = 0; i < plan->n; i++) {
		const int64_t L = produced(plan, st.h, i);
		if (L > 0)
			B200Z_CUDA(cudaMemcpyAsync(dst ? dst[i] : st.hout.p + plan->out_off[(size_t)i], st.dout.p + plan->out_off[(size_t)i], (size_t)L,
			                           cudaMemcpyDeviceToHost, s));
	}
	B200Z_CUDA(cudaStreamSynchronize(s));
	return B200Z_OK;
}

static int pipeline_finish_create(b200z_plan *plan, int wrap, int depth, b200z_pipeline **out) {
	DeviceGuard guard(plan->device);
	if (depth < 1 || depth > 8) {
		b200z_plan_destroy(plan);
		set_error("depth");
		return B200Z_E_ARG;
	}
	b200z_pipeline *p = new b200z_pipeline();
	p->plan = plan;
	p->wrap = wrap;
	p->depth = depth;
	p->slots.resize((size_t)depth);
	int rc = B200Z_OK;
	auto fail = [&](int code) {
		b200z_pipeline_destroy(p);
		return code;
	};
	if (cudaStreamCreateWithFlags(&p->s_up, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&p->s_run, cudaStreamNonBlocking) != cudaSuccess ||
	    cudaStreamCreateWithFlags(&p->s_down, cudaStreamNonBlocking) != cudaSuccess) {
		set_error("cudaStreamCreate failed");
		return fail(B200Z_E_CUDA);
	}
	for (auto &sl : p->slots) {
		if ((rc = sl.ensure(plan, plan->kind == 0))) return fail(rc);
		memset(sl.hin.p, 0, (size_t)plan->in_bytes + 256);
		if (cudaEventCreateWithFlags(&sl.ev_up, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&sl.ev_run, cudaEventDisableTiming) != cudaSuccess) {
			set_error("cudaEventCreate failed");
			return fail(B200Z_E_CUDA);
		}
		// the bytes between the slots of the input blob are never written again: clear them once
		if (cudaMemset(sl.din.p, 0, (size_t)plan->in_bytes + 256) != cudaSuccess) return fail(B200Z_E_CUDA);
	}
	*out = p;
	return B200Z_OK;
}

// ---- host-buffer batch calls: one submit + collect on a cached pipeline of the batch's shape --------------------------
struct PipeKey {
	int device, kind, n, level, strategy, wrap, end_mode;
	std::vector<int64_t> a, b;
	bool operator==(const PipeKey &o) const {
		return device == o.device && kind == o.kind && n == o.n && level == o.level && strategy == o.strategy && wrap == o.wrap &&
		       end_mode == o.end_mode && a == o.a && b == o.b;
	}
};
// Per host thread: the four most recently used shapes of each device keep their plan, staging and device buffers.  A
// pipeline with a batch in flight is not evicted (one _multi call can put two ranges on the same device).
struct PipeCache {
	std::vector<std::pair<PipeKey, b200z_pipeline *>> items; // most recently used first
	~PipeCache() { clear(); }
	b200z_pipeline *find(const PipeKey &k) {
		for (size_t i = 0; i < items.size(); i++)
			if (items[i].first == k) {
				auto it = items[i];
				items.erase(items.begin() + (ptrdiff_t)i);
				items.insert(items.begin(), it);
				return it.second;
			}
		return nullptr;
	}
	void put(PipeKey k, b200z_pipeline *p) {
		const int device = k.device;
		items.insert(items.begin(), std::make_pair(std::move(k), p));
		int same = 0;
		for (size_t i = 0; i < items.size();) {
			if (items[i].first.device == device && ++same > 4 && b200z_pipeline_in_flight(items[i].second) == 0) {
				b200z_pipeline_destroy(items[i].second);
				items.erase(items.begin() + (ptrdiff_t)i);
			} else {
				++i;
			}
		}
	}
	void clear() {
		for (auto &it : items) b200z_pipeline_destroy(it.second);
		items.clear();
	}
};
static thread_local PipeCache g_pipes;

static int multi_batch(int kind, const int32_t *devices, int32_t n_devices, const uint8_t *const *in, const int64_t *in_len, int32_t n, int level,
                       int strategy, int wrap, int end_mode, uint8_t *const *out, const int64_t *out_cap, int64_t *out_len, int64_t *in_used,
                       uint32_t *check, int32_t *status) {
	if (n < 0 || n_devices < 1 || !devices || (n > 0 && (!in || !in_len || !out || !out_cap || !out_len))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const int ndev_all = b200z_device_count();
	for (int d = 0; d < n_devices; d++)
		if (devices[d] < 0 || devices[d] >= ndev_all) {
			set_error("device %d out of range (%d devices)", devices[d], ndev_all);
			return B200Z_E_ARG;
		}
	std::vector<int32_t> first((size_t)n_devices + 1);
	int rc = b200z_partition_by_bytes(in_len, n, n_devices, first.data());
	if (rc) return rc;
	const int saved = t_device;
	std::vector<b200z_pipeline *> pipes((size_t)n_devices, nullptr);
	int result = B200Z_OK;
	for (int d = 0; d < n_devices && result == B200Z_OK; d++) {
		const int a = first[(size_t)d], cnt = first[(size_t)d + 1] - a;
		if (cnt == 0) continue;
		PipeKey key{devices[d], kind, cnt, level, strategy, wrap, end_mode, std::vector<int64_t>(in_len + a, in_len + a + cnt),
		            kind != 0 ? std::vector<int64_t>(out_cap + a, out_cap + a + cnt) : std::vector<int64_t>()};
		b200z_pipeline *p = g_pipes.find(key);
		if (!p) {
			if ((rc = b200z_init(devices[d]))) { result = rc; break; } // (makes the device this thread's current one for the creation)
			rc = kind == 0   ? b200z_deflate_pipeline_create(cnt, in_len + a, level, strategy, wrap, end_mode, 1, &p)
			     : kind == 1 ? b200z_inflate_pipeline_create(cnt, in_len + a, out_cap + a, wrap, 1, &p)
			                 : b200z_lzw_pipeline_create(cnt, in_len + a, out_cap + a, 1, &p);
			if (rc) { result = rc; break; }
			g_pipes.put(std::move(key), p);
		}
		pipes[(size_t)d] = p;
		if ((rc = b200z_pipeline_submit(p, in + a))) result = rc;
	}
	for (int d = 0; d < n_devices; d++) { // everything that was submitted is collected, whatever happened to the others
		b200z_pipeline *p = pipes[(size_t)d];
		if (!p || b200z_pipeline_in_flight(p) == 0) continue;
		const int a = first[(size_t)d];
		rc = b200z_pipeline_collect(p, out + a, out_cap + a, out_len + a, in_used ? in_used + a : nullptr, check ? check + a : nullptr,
		                            status ? status + a : nullptr);
		if (rc && result == B200Z_OK) result = rc;
	}
	t_device = saved;
	if (saved >= 0) cudaSetDevice(saved);
	return result;
}

} // namespace b200z

using namespace b200z;

extern "C" {

int b200z_deflate_pipeline_create(int32_t n, const int64_t *in_len, int level, int strategy, int wrap, int end_mode, int depth,
                                  b200z_pipeline **pipe) {
	if (!pipe) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (level == -1) level = 6;
	if (end_mode == B200Z_END_NONE) {
		set_error("pipelines and batch calls return whole streams: open runs (B200Z_END_NONE) need the deflate plan calls");
		return B200Z_E_UNSUPPORTED;
	}
	b200z_plan *plan = nullptr;
	// gzip: the plan delivers the raw stream and the CRC-32; collect() writes header and trailer (GzipOutputStream.cs:315-375)
	int rc = b200z_deflate_plan_create(n, in_len, level, strategy, wrap == B200Z_WRAP_GZIP ? B200Z_WRAP_RAW_CRC32 : wrap, end_mode, &plan);
	if (rc) return rc;
	return pipeline_finish_create(plan, wrap, depth, pipe);
}

int b200z_inflate_pipeline_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, int wrap, int depth, b200z_pipeline **pipe) {
	if (!pipe) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	b200z_plan *plan = nullptr;
	int rc = b200z_inflate_plan_create(n, comp_len, out_cap, wrap, &plan);
	if (rc) return rc;
	return pipeline_finish_create(plan, wrap, depth, pipe);
}

int b200z_lzw_pipeline_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, int depth, b200z_pipeline **pipe) {
	if (!pipe) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	b200z_plan *plan = nullptr;
	int rc = b200z_lzw_plan_create(n, comp_len, out_cap, &plan);
	if (rc) return rc;
	return pipeline_finish_create(plan, B200Z_WRAP_RAW, depth, pipe);
}

int b200z_pipeline_destroy(b200z_pipeline *p) {
	DeviceGuard guard((p && p->plan) ? p->plan->device : -1);
	if (!p) return B200Z_OK;
	if (p->s_up) cudaStreamSynchronize(p->s_up);
	if (p->s_run) cudaStreamSynchronize(p->s_run);
	if (p->s_down) cudaStreamSynchronize(p->s_down);
	for (auto &sl : p->slots) {
		if (sl.ev_up) cudaEventDestroy(sl.ev_up);
		if (sl.ev_run) cudaEventDestroy(sl.ev_run);
	}
	if (p->s_up) cudaStreamDestroy(p->s_up);
	if (p->s_run) cudaStreamDestroy(p->s_run);
	if (p->s_down) cudaStreamDestroy(p->s_down);
	b200z_plan_destroy(p->plan);
	delete p;
	return B200Z_OK;
}

int32_t b200z_pipeline_in_flight(const b200z_pipeline *p) { return p ? (int32_t)(p->head - p->tail) : 0; }

int b200z_pipeline_submit(b200z_pipeline *p, const uint8_t *const *in) {
	DeviceGuard guard((p && p->plan) ? p->plan->device : -1);
	if (!p || (p->plan->n > 0 && !in)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (p->head - p->tail >= p->depth) {
		set_error("pipeline: %d batches in flight, collect one first", p->depth);
		return B200Z_E_STATE;
	}
	b200z_plan *plan = p->plan;
	const int n = plan->n;
	bool all_pinned = n > 0;
	for (int i = 0; i < n && all_pinned; i++) {
		const int64_t len = plan->in_len[(size_t)i];
		if (len > 0 && !in[i]) {
			set_error("stream %d: null input", i);
			return B200Z_E_ARG;
		}
		if (len > 0 && (i < 4 || (i & 63) == 0)) all_pinned = host_ptr_is_pinned(in[i]); // (sampled: the check is not free)
	}
	b200z_pipeline::Slot &sl = p->slots[(size_t)(p->head % p->depth)];
	int rc = stage_run(plan, sl, in, all_pinned, nullptr, p->s_up, p->s_run, sl.ev_up);
	if (rc) return rc;
	B200Z_CUDA(cudaEventRecord(sl.ev_run, p->s_run));
	++p->head;
	return B200Z_OK;
}

int b200z_pipeline_collect(b200z_pipeline *p, uint8_t *const *out, const int64_t *out_cap, int64_t *out_len, int64_t *in_used,
                           uint32_t *check, int32_t *status) {
	DeviceGuard guard((p && p->plan) ? p->plan->device : -1);
	if (!p || (p->plan->n > 0 && (!out || !out_cap || !out_len))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (p->head == p->tail) {
		set_error("pipeline: nothing submitted");
		return B200Z_E_STATE;
	}
	b200z_plan *plan = p->plan;
	const int n = plan->n;
	b200z_pipeline::Slot &sl = p->slots[(size_t)(p->tail % p->depth)];
	B200Z_CUDA(cudaEventSynchronize(sl.ev_run)); // the run's sizes, statuses and checksums are on the host
	const int wrap = p->wrap;
	int first = B200Z_OK, first_detail = 0;
	int64_t moved = 0;
	if (plan->kind == 0) {
		// ---- deflate: exactly the produced bytes cross PCIe (packed back to back on the device) ----
		const int64_t total = n ? sl.h.poff[n] : 0;
		if (total > 0) B200Z_CUDA(cudaMemcpyAsync(sl.hout.p, sl.dpack.p, (size_t)total, cudaMemcpyDeviceToHost, p->s_down));
		B200Z_CUDA(cudaStreamSynchronize(p->s_down));
		const int hdr = wrap == B200Z_WRAP_ZLIB ? 2 : (wrap == B200Z_WRAP_GZIP ? 10 : 0);
		const int trl = wrap == B200Z_WRAP_ZLIB ? 4 : (wrap == B200Z_WRAP_GZIP ? 8 : 0);
		for (int i = 0; i < n; i++) {
			int st = sl.h.status[i] & 0xFF;
			const int64_t need = sl.h.out_len[i] + hdr + trl;
			if (st == B200Z_OK && need > out_cap[i]) st = B200Z_E_NOMEM;
			out_len[i] = st == B200Z_OK ? need : 0;
			if (status) status[i] = st;
			if (check) check[i] = sl.h.check[i];
			if (in_used) in_used[i] = 0;
			if (st != B200Z_OK && first == B200Z_OK) first = st;
			if (st == B200Z_OK) moved += need;
		}
		host_parallel_for(n, moved, [&](int a, int b) {
			for (int i = a; i < b; i++) {
				if (out_len[i] == 0) continue;
				uint8_t *o = out[i];
				if (wrap == B200Z_WRAP_ZLIB) {
					zlib_header(plan->level, o);
					o += 2;
				} else if (wrap == B200Z_WRAP_GZIP) {
					// GzipOutputStream.GetHeader (:339-375) with MTIME 0 and no FNAME: 1F 8B 08 00 <mtime> 00 FF (trap T15)
					const uint8_t h[10] = {0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF};
					memcpy(o, h, 10);
					o += 10;
				}
				memcpy(o, sl.hout.p + sl.h.poff[i], (size_t)sl.h.out_len[i]);
				o += sl.h.out_len[i];
				const uint32_t a32 = sl.h.check[i];
				if (wrap == B200Z_WRAP_ZLIB) { // Adler32 trailer, big endian (Deflater.cs:509-514)
					o[0] = (uint8_t)(a32 >> 24);
					o[1] = (uint8_t)(a32 >> 16);
					o[2] = (uint8_t)(a32 >> 8);
					o[3] = (uint8_t)a32;
				} else if (wrap == B200Z_WRAP_GZIP) { // GetFooter (:315-337): CRC32, ISIZE = TotalIn & 0xFFFFFFFF, little endian
					const uint32_t isz = (uint32_t)((uint64_t)plan->in_len[(size_t)i] & 0xFFFFFFFFull);
					for (int k = 0; k < 4; k++) o[k] = (uint8_t)(a32 >> (8 * k));
					for (int k = 0; k < 4; k++) o[4 + k] = (uint8_t)(isz >> (8 * k));
				}
			}
		});
	} else {
		// ---- inflate and LZW: every stream's produced bytes; straight into the caller's buffers when CUDA knows them as
		// pinned.  An LZW stream that needs more than its capacity reports B200Z_E_NOMEM and the size it needs in out_len. ----
		bool all_pinned = n > 0;
		for (int i = 0; i < n && all_pinned; i++)
			if (produced(plan, sl.h, i) > 0 && (i < 4 || (i & 63) == 0)) all_pinned = host_ptr_is_pinned(out[i]);
		int rc = streams_down(plan, sl, all_pinned ? out : nullptr, p->s_down);
		if (rc) return rc;
		for (int i = 0; i < n; i++) moved += produced(plan, sl.h, i);
		if (!all_pinned)
			host_parallel_for(n, moved, [&](int a, int b) {
				for (int i = a; i < b; i++)
					if (produced(plan, sl.h, i) > 0) memcpy(out[i], sl.hout.p + plan->out_off[(size_t)i], (size_t)produced(plan, sl.h, i));
			});
		for (int i = 0; i < n; i++) {
			const int st = sl.h.status[i];
			out_len[i] = sl.h.out_len[i];
			if (in_used) in_used[i] = sl.h.in_used[i];
			if (status) status[i] = st;
			if (check) check[i] = wrap != B200Z_WRAP_RAW || plan->kind == 2 ? sl.h.check[i] : 0u; // (LZW: the message's numbers)
			if ((st & 0xFF) != B200Z_OK && first == B200Z_OK) {
				first = st & 0xFF;
				first_detail = (st >> 8) & 0xFF;
			}
		}
	}
	++p->tail;
	if (first == B200Z_E_DATA && plan->kind == 1) set_error("%s", inflate_detail_msg(first_detail)); // the reference's exception message
	else if (plan->kind == 2 && (first == B200Z_E_DATA || first == B200Z_E_INTERNAL)) {
		for (int i = 0; i < n; i++)
			if ((sl.h.status[i] & 0xFF) == first) {
				set_error("%s", lzw_detail_msg(sl.h.status[i], sl.h.check[i]).c_str());
				break;
			}
	}
	else if (first != B200Z_OK) set_error("stream failed with status %d", first);
	return first;
}

int b200z_release_cached(void) { // frees what the host-buffer batch calls of this thread keep between calls
	g_pipes.clear();
	return B200Z_OK;
}

// The single-device batch calls are the _multi calls on the calling thread's device.  ensure_init() comes first: without a
// device they fail with B200Z_E_CUDA, not with the _multi calls' device range check.
int b200z_deflate_batch(const uint8_t *const *in, const int64_t *in_len, int32_t n, int level, int strategy, int wrap,
                        int end_mode, uint8_t *const *out, const int64_t *out_cap, int64_t *out_len, uint32_t *check,
                        int32_t *status) {
	int rc = ensure_init();
	if (rc) return rc;
	const int32_t device = current_device();
	return b200z_deflate_batch_multi(&device, 1, in, in_len, n, level, strategy, wrap, end_mode, out, out_cap, out_len, check, status);
}

int b200z_inflate_batch(const uint8_t *const *in, const int64_t *in_len, int32_t n, int wrap, uint8_t *const *out,
                        const int64_t *out_cap, int64_t *out_len, int64_t *in_used, uint32_t *check, int32_t *status) {
	int rc = ensure_init();
	if (rc) return rc;
	const int32_t device = current_device();
	return b200z_inflate_batch_multi(&device, 1, in, in_len, n, wrap, out, out_cap, out_len, in_used, check, status);
}

int b200z_lzw_batch(const uint8_t *const *in, const int64_t *in_len, int32_t n, uint8_t *const *out, const int64_t *out_cap,
                    int64_t *out_len, int64_t *in_used, uint32_t *value, int32_t *status) {
	int rc = ensure_init();
	if (rc) return rc;
	const int32_t device = current_device();
	return b200z_lzw_batch_multi(&device, 1, in, in_len, n, out, out_cap, out_len, in_used, value, status);
}

// ---- one host thread, several GPUs ----------------------------------------------------------------------------------
// The streams of a batch are independent (a fresh Deflater / Inflater each): they are cut into contiguous ranges of
// about equal bytes (SURVEY.md 8e), every range goes to one device's pipeline, all submits are issued before the first
// collect -- the devices work at the same time, the calling thread only stages and waits.
int b200z_device_count(void) {
	int cnt = 0;
	if (cudaGetDeviceCount(&cnt) != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return cnt;
}

int b200z_partition_by_bytes(const int64_t *len, int32_t n, int32_t parts, int32_t *first) {
	if (n < 0 || parts < 1 || !first || (n > 0 && !len)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int64_t total = 0;
	for (int i = 0; i < n; i++) total += len[i] > 0 ? len[i] : 0;
	// part r starts at the first stream whose cumulative start offset is >= floor(r T / R)
	int32_t i = 0;
	int64_t start = 0; // cumulative start of stream i
	first[0] = 0;
	for (int r = 1; r < parts; r++) {
		const int64_t cut = (int64_t)(((__int128)total * r) / parts);
		while (i < n && start < cut) {
			start += len[i] > 0 ? len[i] : 0;
			++i;
		}
		first[r] = i;
	}
	first[parts] = n;
	return B200Z_OK;
}

int b200z_deflate_batch_multi(const int32_t *devices, int32_t n_devices, const uint8_t *const *in, const int64_t *in_len, int32_t n, int level,
                              int strategy, int wrap, int end_mode, uint8_t *const *out, const int64_t *out_cap, int64_t *out_len,
                              uint32_t *check, int32_t *status) {
	if (level == -1) level = 6;
	return multi_batch(0, devices, n_devices, in, in_len, n, level, strategy, wrap, end_mode, out, out_cap, out_len, nullptr, check, status);
}

int b200z_inflate_batch_multi(const int32_t *devices, int32_t n_devices, const uint8_t *const *in, const int64_t *in_len, int32_t n, int wrap,
                              uint8_t *const *out, const int64_t *out_cap, int64_t *out_len, int64_t *in_used, uint32_t *check,
                              int32_t *status) {
	return multi_batch(1, devices, n_devices, in, in_len, n, 0, 0, wrap, 0, out, out_cap, out_len, in_used, check, status);
}

int b200z_lzw_batch_multi(const int32_t *devices, int32_t n_devices, const uint8_t *const *in, const int64_t *in_len, int32_t n,
                          uint8_t *const *out, const int64_t *out_cap, int64_t *out_len, int64_t *in_used, uint32_t *value, int32_t *status) {
	return multi_batch(2, devices, n_devices, in, in_len, n, 0, 0, B200Z_WRAP_RAW, 0, out, out_cap, out_len, in_used, value, status);
}

} // extern "C"
