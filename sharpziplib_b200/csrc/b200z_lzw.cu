// b200z_lzw.cu -- LZW (.Z, Unix compress) decompression: LzwInputStream (Lzw/LzwInputStream.cs) for a batch of independent
// streams.  Every code after the first of a stream expands to the string of an earlier code plus one byte, so a stream is a
// forest of codes: a literal is a root, any other code is a child of the code whose string it extends.  The kernels
//   k_lzw_scan    one warp per stream, 32 codes per step: header, code positions (width growth and padding, CLEAR), validation, and for
//                 every code its parent and the code whose first byte ends its string
//   k_lzw_jump    pointer jumping over the parents (17 rounds cover the longest string, 65281 bytes): depth and root
//   k_lzw_last    string length and last byte of every code
//   k_lzw_offsets one block per stream: output offsets (int64), out_len, NOMEM
//   k_lzw_emit    one thread per code: walks its ancestors and writes its string back to front
// No byte is decoded on the host.
#include <algorithm>

#include "b200z_internal.cuh"

namespace b200z {


constexpr int kJumpRounds = 17; // 2^17 > the deepest code: 65536 - 256 entries + the KwK byte

// One code of a stream.  par: parent code (index in the stream), or -1 - byte for a literal; src: the code whose first byte is
// this code's last byte (a literal's own byte is its last).
struct __align__(8) LzwCode {
	int32_t par, src;
};

struct LzwStream {
	int64_t ncodes;  // data codes in front of the first bad one (CLEARs are not codes here)
	int64_t in_used; // bytes of the stream up to the last code read
	int32_t epochs;  // CLEARs + 1
	int32_t status;  // code | detail << 8
	uint32_t value;  // the numbers the reference's message quotes (INTEGRATION.md §2)
	int32_t pad_;
};

// the stream whose code slots hold global code i: code_base has n + 1 entries
__device__ __forceinline__ int stream_of(const int64_t *__restrict__ code_base, int n, int64_t i) {
	int lo = 0, hi = n - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (code_base[mid] <= i) lo = mid;
		else hi = mid - 1;
	}
	return lo;
}

__device__ __forceinline__ uint32_t byte_at(const uint8_t *p, int64_t len, int64_t i) { return i < len ? p[i] : 0u; }

// One warp per stream.  Between two width changes the codes are nb bits apart and freeEnt grows by one per code, so the
// warp reads 32 codes per step, each lane at a position that follows from its index; a ballot finds the first code that
// ends the step (CLEAR, a bad code, or no more bits), and the codes in front of it are written.
__global__ void __launch_bounds__(128)
    k_lzw_scan(int n, const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
               const int64_t *__restrict__ code_base, LzwCode *__restrict__ codes, LzwStream *__restrict__ st) {
	const int lane = threadIdx.x & 31;
	const int s = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
	if (s >= n) return; // (the whole warp)
	const uint8_t *p = in + in_off[s];
	const int64_t L = in_len[s];
	LzwCode *cd = codes + code_base[s];
	LzwStream r{};
	r.epochs = 1;
	auto fail = [&](int code, int detail, uint32_t value) {
		r.status = code | detail << 8;
		r.value = value;
	};
	// ParseHeader (:336-387): one Read of 3 bytes, a short read leaves zeros
	const uint32_t h0 = byte_at(p, L, 0), h1 = byte_at(p, L, 1), h2 = byte_at(p, L, 2);
	const int max_bits = (int)(h2 & 0x1F);
	const bool block = (h2 & 0x80) != 0;
	if (h0 != 0x1F || h1 != 0x9D) fail(B200Z_E_DATA, 32, h0 << 8 | h1);
	else if (max_bits > 16) fail(B200Z_E_DATA, 33, (uint32_t)max_bits);
	else if (h2 & 0x60) fail(B200Z_E_DATA, 34, 0);
	else if (max_bits < 8) fail(B200Z_E_INTERNAL, 1, (uint32_t)max_bits); // tabSuffix[255] in a table of 1 << maxBits
	if (r.status) {
		if (lane == 0) st[s] = r;
		return;
	}
	const uint8_t *d = p + 3;
	const int64_t dl = L > 3 ? L - 3 : 0, dbits = 8 * dl;
	const int max_max = 1 << max_bits;
	// warp-uniform state
	int nb = 9, max_code = 511, free_ent = block ? 257 : 256;
	int64_t bit = 0, group = 0; // position; where the current width began (the padding counts from there)
	int64_t k = 0;              // data codes so far
	int64_t base = 0;           // the entry c of this epoch was defined by code base + c
	int old = -1;               // oldCode: not reset by a CLEAR
	auto read = [&](int64_t b) {
		const int64_t q = b >> 3;
		const uint32_t w = byte_at(d, dl, q) | byte_at(d, dl, q + 1) << 8 | byte_at(d, dl, q + 2) << 16;
		return (int)((w >> (b & 7)) & ((1u << nb) - 1));
	};
	auto pad = [&] { // to a whole group of nb-bit codes; ResetBuf copies a negative length when that is past the data
		const int64_t g = 8 * nb;
		bit = group + (bit - group + g - 1) / g * g;
		group = bit;
		if ((bit >> 3) > dl) fail(B200Z_E_INTERNAL, 2, 0);
		return r.status == 0;
	};
	for (;;) {
		if (bit + nb > dbits) break; // a code is read only when all its bits are there
		if (free_ent > max_code) {
			if (!pad()) break;
			nb++;
			max_code = nb == max_bits ? max_max : (1 << nb) - 1;
			continue;
		}
		if (old == -1) { // the stream's first code defines nothing
			const int c = read(bit);
			bit += nb;
			if (c >= 256) {
				fail(B200Z_E_DATA, 35, (uint32_t)c);
				break;
			}
			if (lane == 0) cd[k] = LzwCode{-1 - c, 0};
			base = 1 - free_ent;
			old = c;
			r.in_used = 3 + ((bit + 7) >> 3);
			++k;
			continue;
		}
		// codes left at this width: freeEnt passes maxCode after m more codes (never when the table fills first)
		const int64_t m = max_max > max_code ? (int64_t)max_code - free_ent + 1 : INT64_MAX;
		const int64_t pb = bit + (int64_t)lane * nb;
		const bool have = lane < m && pb + nb <= dbits;
		const int c = have ? read(pb) : 0;
		// freeEnt when this code is read: it grows up to maxMaxCode (a block-mode 8-bit stream starts above it, at 257)
		const int fe = free_ent >= max_max ? free_ent : (free_ent + lane < max_max ? free_ent + lane : max_max);
		int prev = __shfl_up_sync(0xffffffffu, c, 1);
		if (lane == 0) prev = old;
		const bool clear = c == 256 && block;
		const bool bad = c > fe || (c == fe && prev >= max_max); // (KwK on a KwK in a table of 256: tabSuffix[oldCode])
		const unsigned stop = __ballot_sync(0xffffffffu, !have || clear || bad);
		const int t = stop ? __ffs(stop) - 1 : 32; // codes in front of the first that ends the step
		if (lane < t) {
			LzwCode e;
			if (c < 256) {
				e = LzwCode{-1 - c, 0};
			} else if (c < fe) {
				const int64_t def = base + c; // the code that defined entry c; the entry is that code's predecessor + a byte
				e = LzwCode{(int32_t)(def - 1), (int32_t)def};
			} else {
				e = LzwCode{(int32_t)(k + lane - 1), (int32_t)(k + lane - 1)}; // KwK: the previous string plus its first byte
			}
			cd[k + lane] = e;
		}
		if (t > 0) {
			old = __shfl_sync(0xffffffffu, c, t - 1);
			bit += (int64_t)t * nb;
			k += t;
			if (free_ent < max_max) free_ent = free_ent + t < max_max ? free_ent + t : max_max;
			r.in_used = 3 + ((bit + 7) >> 3);
		}
		if (t == 32 || !((__ballot_sync(0xffffffffu, have) >> t) & 1)) continue; // (a width change or the end: the loop top)
		const int cs = __shfl_sync(0xffffffffu, c, t);
		const bool clear_s = __shfl_sync(0xffffffffu, clear, t);
		bit += nb;
		if (clear_s) {
			if (!pad()) break;
			nb = 9;
			max_code = 511;
			free_ent = 256;
			base = k - 256;
			++r.epochs;
			continue;
		}
		if (cs > free_ent) fail(B200Z_E_DATA, 36, (uint32_t)cs << 16 | (uint32_t)free_ent);
		else fail(B200Z_E_INTERNAL, 4, 0);
		break;
	}
	r.ncodes = k;
	if (lane == 0) st[s] = r;
}

// pd: (.x the ancestor reached so far, .y how many generations up it is); codes past a stream's last valid one are roots.
// Round 0 reads the parents from the codes.
__global__ void __launch_bounds__(256)
    k_lzw_jump(int64_t total, int n, const int64_t *__restrict__ code_base, const LzwStream *__restrict__ st,
               const LzwCode *__restrict__ codes, const int2 *__restrict__ pd_in, int2 *__restrict__ pd_out, int first) {
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
		const int s = stream_of(code_base, n, i);
		const int64_t b = code_base[s];
		const int32_t j = (int32_t)(i - b);
		if (j >= st[s].ncodes) {
			pd_out[i] = make_int2(j, 0);
			continue;
		}
		int2 v, u;
		if (first) {
			const int32_t par = codes[i].par;
			v = par < 0 ? make_int2(j, 0) : make_int2(par, 1);
			const int32_t pp = codes[b + v.x].par;
			u = pp < 0 ? make_int2(v.x, 0) : make_int2(pp, 1);
		} else {
			v = pd_in[i];
			u = pd_in[b + v.x];
		}
		pd_out[i] = make_int2(u.x, v.y + u.y);
	}
}

__global__ void __launch_bounds__(256)
    k_lzw_last(int64_t total, int n, const int64_t *__restrict__ code_base, const LzwStream *__restrict__ st,
               const LzwCode *__restrict__ codes, const int2 *__restrict__ pd, int64_t *__restrict__ len, uint8_t *__restrict__ last,
               unsigned int *__restrict__ longest) {
	unsigned int mx = 0;
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
		const int s = stream_of(code_base, n, i);
		const int64_t b = code_base[s];
		if (i - b >= st[s].ncodes) continue;
		const LzwCode c = codes[i];
		const int2 v = pd[i];
		const int32_t lit = c.par < 0 ? c.par : codes[b + pd[b + c.src].x].par; // the root of src is a literal
		last[i] = (uint8_t)(-1 - lit);
		len[i] = v.y + 1;
		mx = mx > (unsigned int)(v.y + 1) ? mx : (unsigned int)(v.y + 1);
	}
	for (int o = 16; o > 0; o >>= 1) {
		const unsigned int t = __shfl_xor_sync(0xffffffffu, mx, o);
		mx = mx > t ? mx : t;
	}
	if ((threadIdx.x & 31) == 0 && mx) atomicMax(longest, mx);
}

// one block per stream: exclusive scan of the string lengths in place, then out_len and the final status
__global__ void __launch_bounds__(1024)
    k_lzw_offsets(const int64_t *__restrict__ code_base, LzwStream *__restrict__ st, int64_t *__restrict__ len,
                  const int64_t *__restrict__ out_cap, int64_t *__restrict__ out_len, int32_t *__restrict__ status,
                  uint32_t *__restrict__ value, int64_t *__restrict__ in_used) {
	__shared__ int64_t s_part[32];
	__shared__ int64_t s_carry;
	const int s = blockIdx.x;
	const int64_t nc = st[s].ncodes;
	int64_t *l = len + code_base[s];
	if (threadIdx.x == 0) s_carry = 0;
	__syncthreads();
	for (int64_t base = 0; base < nc; base += 1024) {
		const int64_t i = base + threadIdx.x;
		const int64_t v = i < nc ? l[i] : 0;
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
		if (i < nc) l[i] = carry + woff + incl - v;
		__syncthreads();
		if (threadIdx.x == 1023) s_carry = carry + woff + incl;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		const int64_t total = s_carry;
		LzwStream r = st[s];
		if (total > out_cap[s]) { // .Z has no size field: report what the stream needs
			r.status = B200Z_E_NOMEM;
			st[s].status = r.status;
		}
		out_len[s] = total;
		status[s] = r.status;
		if (value) value[s] = r.value;
		if (in_used) in_used[s] = r.in_used;
	}
}

__global__ void __launch_bounds__(256)
    k_lzw_emit(int64_t total, int n, const int64_t *__restrict__ code_base, const LzwStream *__restrict__ st,
               const LzwCode *__restrict__ codes, const int64_t *__restrict__ off, const uint8_t *__restrict__ last,
               const int2 *__restrict__ pd, const int64_t *__restrict__ out_off, uint8_t *__restrict__ out) {
	for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
		const int s = stream_of(code_base, n, i);
		const int64_t b = code_base[s];
		if (i - b >= st[s].ncodes || (st[s].status & 0xFF) == B200Z_E_NOMEM) continue;
		uint8_t *o = out + out_off[s] + off[i];
		int64_t j = i;
		for (int k = pd[i].y; k >= 0; k--) { // the string is the last bytes of the code's ancestors, root first
			o[k] = last[j];
			j = b + codes[j].par;
		}
	}
}

// The plan of kind 2: n LZW streams of comp_len bytes (header included) decoding into at most out_cap bytes each.
struct LzwPlan : b200z_plan {
	int64_t codes = 0; // code slots: every stream gets room for one code per 9 bits
	std::vector<int64_t> code_base;
	Slot<int64_t> o_code_base;
	Slot<LzwCode> o_codes;
	Slot<LzwStream> o_st;
	Slot<int2> o_pd0, o_pd1;
	Slot<int64_t> o_len;
	Slot<uint8_t> o_last;
	Slot<unsigned int> o_longest;
};

int lzw_plan_create(int32_t n, const int64_t *comp_len, const int64_t *out_cap, b200z_plan **out) {
	for (int i = 0; i < n; i++)
		if (comp_len[i] < 0 || comp_len[i] > 0x7FFFFFFFll || out_cap[i] < 0) {
			set_error("stream %d: compressed length %lld (0..2^31-1), capacity %lld", i, (long long)comp_len[i], (long long)out_cap[i]);
			return B200Z_E_ARG;
		}
	LzwPlan *p = new LzwPlan();
	p->kind = 2;
	p->device = current_device();
	p->n = n;
	p->in_len.assign(comp_len, comp_len + n);
	p->out_cap.assign(out_cap, out_cap + n);
	p->in_off.resize((size_t)n);
	p->out_off.resize((size_t)n);
	p->code_base.resize((size_t)n + 1);
	for (int i = 0; i < n; i++) {
		p->in_off[(size_t)i] = p->in_bytes;
		p->in_bytes = align_up(p->in_bytes + comp_len[i], kAlign);
		p->out_off[(size_t)i] = p->out_bytes;
		p->out_bytes = align_up(p->out_bytes + out_cap[i] + 16, kAlign);
		p->code_base[(size_t)i] = p->codes;
		p->codes += comp_len[i] > 3 ? (comp_len[i] - 3) * 8 / 9 : 0;
	}
	p->code_base[(size_t)n] = p->codes;
	p->upload_streams(p->in_off, p->in_len, 0);
	p->o_code_base = p->ws.upload(p->code_base);
	p->o_codes = p->ws.reserve<LzwCode>(p->codes);
	p->o_st = p->ws.reserve<LzwStream>(n);
	p->o_pd0 = p->ws.reserve<int2>(p->codes);
	p->o_pd1 = p->ws.reserve<int2>(p->codes);
	p->o_len = p->ws.reserve<int64_t>(p->codes);
	p->o_last = p->ws.reserve<uint8_t>(p->codes);
	p->o_longest = p->ws.reserve<unsigned int>(1);
	p->launches = 3 + kJumpRounds + 2;
	const int rc = p->ws.alloc();
	if (rc) {
		delete p;
		return rc;
	}
	*out = p;
	return B200Z_OK;
}

int lzw_plan_run(b200z_plan *bp, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status, uint32_t *d_value,
                 int64_t *d_in_used, cudaStream_t s) {
	LzwPlan *p = static_cast<LzwPlan *>(bp);
	if (p->n == 0) return B200Z_OK;
	p->ev_used = 0;
	const Arena &w = p->ws;
	int sms = 132;
	B200Z_CUDA(sm_count(&sms));
	const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((p->codes + 255) / 256, (int64_t)sms * 8));
	B200Z_CUDA(cudaMemsetAsync(w.at(p->o_longest), 0, 4, s));
	p->mark(s, "k_lzw_scan");
	k_lzw_scan<<<(p->n + 3) / 4, 128, 0, s>>>(p->n, d_in, w.at(p->o_in_off), w.at(p->o_in_len), w.at(p->o_code_base), w.at(p->o_codes),
	                                               w.at(p->o_st));
	B200Z_CUDA(cudaGetLastError());
	p->mark(s, "k_lzw_jump");
	int2 *a = w.at(p->o_pd0), *b = w.at(p->o_pd1);
	if (p->codes > 0)
		for (int r = 0; r < kJumpRounds; r++) {
			k_lzw_jump<<<grid, 256, 0, s>>>(p->codes, p->n, w.at(p->o_code_base), w.at(p->o_st), w.at(p->o_codes), a, b, r == 0);
			std::swap(a, b);
		}
	B200Z_CUDA(cudaGetLastError());
	p->mark(s, "k_lzw_last");
	if (p->codes > 0)
		k_lzw_last<<<grid, 256, 0, s>>>(p->codes, p->n, w.at(p->o_code_base), w.at(p->o_st), w.at(p->o_codes), a, w.at(p->o_len),
		                                w.at(p->o_last), w.at(p->o_longest));
	p->mark(s, "k_lzw_offsets");
	k_lzw_offsets<<<p->n, 1024, 0, s>>>(w.at(p->o_code_base), w.at(p->o_st), w.at(p->o_len), w.at(p->o_out_cap), d_out_len, d_status,
	                                    d_value, d_in_used);
	B200Z_CUDA(cudaGetLastError());
	p->mark(s, "k_lzw_emit");
	if (p->codes > 0)
		k_lzw_emit<<<grid, 256, 0, s>>>(p->codes, p->n, w.at(p->o_code_base), w.at(p->o_st), w.at(p->o_codes), w.at(p->o_len),
		                                w.at(p->o_last), a, p->dev_out_off(), d_out);
	B200Z_CUDA(cudaGetLastError());
	p->mark(s, "end");
	return B200Z_OK;
}

// epochs, codes (summed over the streams) and the longest string of the last run
int lzw_plan_stats(b200z_plan *bp, uint32_t *v, int32_t cap, cudaStream_t s) {
	LzwPlan *p = static_cast<LzwPlan *>(bp);
	std::vector<LzwStream> st((size_t)p->n);
	unsigned int longest = 0;
	if (p->n) B200Z_CUDA(cudaMemcpyAsync(st.data(), p->ws.at(p->o_st), sizeof(LzwStream) * p->n, cudaMemcpyDeviceToHost, s));
	B200Z_CUDA(cudaMemcpyAsync(&longest, p->ws.at(p->o_longest), 4, cudaMemcpyDeviceToHost, s));
	B200Z_CUDA(cudaStreamSynchronize(s));
	uint64_t epochs = 0, codes = 0;
	for (const auto &r : st) epochs += (uint32_t)r.epochs, codes += (uint64_t)r.ncodes;
	const uint32_t vals[3] = {(uint32_t)std::min<uint64_t>(epochs, 0xFFFFFFFFu), (uint32_t)std::min<uint64_t>(codes, 0xFFFFFFFFu), longest};
	for (int i = 0; i < cap && i < 3; i++) v[i] = vals[i];
	return B200Z_OK;
}

} // namespace b200z
