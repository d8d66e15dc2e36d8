// model.cpp -- TEST INFRASTRUCTURE.  Serial host execution of the *kernel decomposition* in
// sharpziplib_b200/csrc/b200z_core.cuh (the very same __host__ __device__ functions the sm_90a kernels call),
// so the exactness of the parallel reformulation can be checked against the oracle in the CPU-only test tier.
// It is not a fallback: the product library never links it.
#include "b200z_core.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace b200z;

namespace {

// K1 as the kernel does it: 32 positions per step, a 16-bit head table relative to a sliding base.
void model_links(const uint8_t *data, uint32_t n, std::vector<uint16_t> &link, uint32_t H = 0, const uint8_t *hmask = nullptr) {
	link.assign(n, 0);
	std::vector<uint16_t> head(32768, 0);
	uint32_t winbase = 0; // head entry v > 0 means position winbase + v - 1
	for (uint32_t base = 0; base < n; base += 32) {
		// re-base so that every stored value stays within 16 bits
		while (base + 32 - winbase > 65535) {
			for (auto &v : head) v = v > 32768 ? (uint16_t)(v - 32768) : 0;
			winbase += 32768;
		}
		uint32_t h[32];
		bool valid[32];
		for (int l = 0; l < 32; l++) {
			uint32_t p = base + l;
			valid[l] = p + 2 < n;
			if (p < H) valid[l] = hmask ? hmask[p] == 0 : p + 2 < H;
			h[l] = valid[l] ? hash3(data[p], data[p + 1], data[p + 2]) : 0xFFFFFFFFu;
		}
		uint32_t q[32];
		for (int l = 0; l < 32; l++) {
			q[l] = 0xFFFFFFFFu;
			if (!valid[l]) continue;
			int lower = -1;
			for (int k = 0; k < l; k++)
				if (valid[k] && h[k] == h[l]) lower = k;
			if (lower >= 0) q[l] = base + lower;
			else if (head[h[l]]) q[l] = winbase + head[h[l]] - 1;
		}
		for (int l = 0; l < 32; l++) {
			if (!valid[l]) continue;
			bool top = true;
			for (int k = l + 1; k < 32; k++)
				if (valid[k] && h[k] == h[l]) top = false;
			if (top) head[h[l]] = (uint16_t)(base + l - winbase + 1);
			uint32_t p = base + l;
			if (q[l] != 0xFFFFFFFFu && p - q[l] <= (uint32_t)kMaxDist) link[p] = (uint16_t)(p - q[l]);
		}
	}
}

struct Writer { // what the emit kernel does with atomicOr on zeroed 32-bit words
	std::vector<uint32_t> w;
	void put(uint64_t bitpos, uint64_t bits, int nbits) {
		while (nbits > 0) {
			uint64_t idx = bitpos >> 5;
			int sh = (int)(bitpos & 31);
			int take = 32 - sh < nbits ? 32 - sh : nbits;
			if (w.size() <= idx) w.resize(idx + 1, 0);
			w[idx] |= (uint32_t)((bits & ((take == 64 ? 0 : (1ull << take)) - 1)) << sh);
			bits >>= take;
			bitpos += take;
			nbits -= take;
		}
	}
};

} // namespace

// History form (b200z_deflate_plan_create_ex): data = H history bytes + the segment, n = both; abs_bias = pos_base - H;
// the bits start at bit_base; end_mode 0 finish / 2 flush (stream stays open); *outbits = total bits (bit_base included)
// sched: the segment's SetInput schedule (cum[i] = bytes after the first i + 1 calls; nchunks 0 = one call); state: the
// engine state of levels 0-4 between segments (kFastStateBytes: head[], prev[], FastCarry / StoredCarry), read when cont != 0
// and written at the end -- what b200z_history.engine_state / stored_state carry for the kernels
struct ModelSched {
	const uint32_t *cum = nullptr;
	int nchunks = 0;
	uint8_t *state = nullptr;
	int cont = 0;
	int busy_last = 1; // 0: Flush() / Finish() right behind the last SetInput, no Deflate() call in between
};
static int model_run(const uint8_t *data, uint32_t n, uint32_t H, uint32_t abs_bias, uint32_t bit_base, const uint8_t *hmask,
                     int level, int strategy, int flush_then_finish, int flush_only, uint8_t *out, uint64_t cap, uint64_t *outlen,
                     uint64_t *outbits, const ModelSched &ms = ModelSched());

extern "C" int model_deflate(const uint8_t *data, uint32_t n, int level, int strategy, int flush_then_finish,
                             uint8_t *out, uint64_t cap, uint64_t *outlen) {
	uint64_t bits;
	return model_run(data, n, 0, 0, 0, nullptr, level, strategy, flush_then_finish, 0, out, cap, outlen, &bits);
}

extern "C" int model_deflate_ex(const uint8_t *data, uint32_t n, uint32_t hist, uint32_t pos_base, uint32_t bit_base,
                                const uint8_t *hmask, int level, int strategy, int end_mode, uint8_t *out, uint64_t cap,
                                uint64_t *outbits) {
	uint64_t len;
	return model_run(data, n, hist, pos_base - hist, bit_base, hmask, level, strategy, 0, end_mode == 2, out, cap, &len, outbits);
}

extern "C" int model_state_bytes() { return kFastStateBytes; }

extern "C" int model_deflate_ex2(const uint8_t *data, uint32_t n, uint32_t hist, uint32_t pos_base, uint32_t bit_base,
                                 const uint8_t *hmask, int level, int strategy, int end_mode, const uint32_t *cum, int nchunks,
                                 int busy_last, uint8_t *state, int cont, uint8_t *out, uint64_t cap, uint64_t *outbits) {
	uint64_t len;
	ModelSched ms;
	ms.cum = cum;
	ms.nchunks = nchunks;
	ms.state = state;
	ms.cont = cont;
	ms.busy_last = busy_last;
	return model_run(data, n, hist, pos_base - hist, bit_base, hmask, level, strategy, 0, end_mode == 2, out, cap, &len, outbits, ms);
}

static int model_run(const uint8_t *data, uint32_t n, uint32_t H, uint32_t abs_bias, uint32_t bit_base, const uint8_t *hmask,
                     int level, int strategy, int flush_then_finish, int flush_only, uint8_t *out, uint64_t cap, uint64_t *outlen,
                     uint64_t *outbits, const ModelSched &ms) {
	LevelParams lp = level_params(level);
	*outbits = 0;
	std::vector<uint32_t> syms;
	std::vector<uint32_t> blk_start(n / kBlockSyms + 3, 0), blk_ptop(n / kBlockSyms + 3, 0);
	size_t nblocks = 0;
	uint32_t total = 0;
	if (lp.func == 0) {
		// level 0: stored blocks only (each block: 3 header bits, pad, LEN, ~LEN, bytes)
		Writer W0;
		uint64_t bp = 0;
		StoredCarry cin, cout;
		if (ms.cont) std::memcpy(&cin, ms.state, sizeof cin);
		stored_run(n - H, ms.cont ? 0 : H, flush_then_finish ? 1 : (flush_only ? 2 : 0), [&](uint32_t start, uint32_t len, bool last) {
			W0.put(bp, last ? 1 : 0, 3);
			bp = (bp + 3 + 7) & ~7ull;
			W0.put(bp, len & 0xFFFF, 16);
			W0.put(bp + 16, (~len) & 0xFFFF, 16);
			bp += 32;
			for (uint32_t i = 0; i < len; i++, bp += 8) W0.put(bp, data[start + i], 8);
		}, ms.cum, ms.nchunks, ms.cont ? &cin : nullptr, &cout, ms.cont ? abs_bias : 0, ms.busy_last != 0);
		if (ms.state) std::memcpy(ms.state, &cout, sizeof cout);
		*outbits = bp;
		uint64_t nb0 = (bp + 7) >> 3;
		if (nb0 > cap) return 102;
		W0.w.resize((nb0 + 3) / 4 + 1, 0);
		std::memcpy(out, W0.w.data(), nb0);
		*outlen = nb0;
		return 0;
	}
	std::vector<uint16_t> link;
	std::vector<uint32_t> tabA, tabB;
	if (lp.func == 1) {
		// levels 1-4: the serial DeflateFast emulation (what k_fast runs, one thread per stream)
		std::vector<uint16_t> head(32768, 0), prev(32768, 0);
		FastEngine fe;
		if (ms.cont) {
			// k_fast: tables and scalars come back from the state buffer the previous segment's run filled
			FastCarry c;
			std::memcpy(head.data(), ms.state, 65536);
			std::memcpy(prev.data(), ms.state + 65536, 65536);
			std::memcpy(&c, ms.state + 131072, sizeof c);
			fe_load(fe, c, data, n, H, head.data(), prev.data());
		} else {
			fe_init(fe, data, n, head.data(), prev.data());
			fe_set_dictionary(fe, H);
		}
		blk_start.assign(n / kBlockSyms + 3, 0);
		fe_run(fe, lp, strategy, (flush_then_finish || flush_only) ? 2 : 0, [&](uint32_t sym) { syms.push_back(sym); },
		       [&](uint32_t start, bool ok, bool last) {
			       (void)last;
			       blk_start[nblocks] = start;
			       blk_ptop[nblocks] = ok ? 0xFFFFFFFEu : 0xFFFFFFFFu;
			       ++nblocks;
		       }, ms.cum, ms.nchunks, ms.busy_last != 0);
		if (ms.state) {
			FastCarry c;
			fe_save(fe, c);
			std::memcpy(ms.state, head.data(), 65536);
			std::memcpy(ms.state + 65536, prev.data(), 65536);
			std::memcpy(ms.state + 131072, &c, sizeof c);
		}
		total = (uint32_t)syms.size();
		goto emit_blocks;
	}
	model_links(data, n, link, H, hmask);
	// K2: every position of the segment (history positions are candidates only)
	tabA.assign(n, 0);
	tabB.assign(n, 0);
	for (uint32_t p = H; p < n; p++) match_search(data, link.data(), 0u, p, n, lp, tabA[p], tabB[p], abs_bias);
	blk_start[0] = H;
	{
	// K3 as k_parse does it: rounds of 32 segments x kSeg positions; every lane parses its segment speculatively from a
	// clean state, entries are handed lane -> lane until nothing changes, then a final pass emits at prefix-summed offsets
	const uint32_t kSeg = 64, kRound = 32 * kSeg;
	auto tabf = [&](uint32_t p, uint32_t &a, uint32_t &b) { a = tabA[p]; b = tabB[p]; };
	auto bytef = [&](uint32_t q) { return (uint32_t)data[q]; };
	auto slowf = [&](uint32_t p, uint32_t m0, uint32_t budget) { return match_search_above(data, link.data(), p, n, m0, budget, abs_bias); };
	ParseCarry carry;
	parse_init(carry.st);
	carry.st.p = H;
	carry.last_top = H;
	int max_iters = 0;
	long sum_iters = 0, n_rounds = 0;
	for (uint32_t base = 0; base < n; base += kRound) {
		ParseCarry entry[32], ex[32];
		uint32_t cnt[32];
		bool changed[32];
		for (int l = 0; l < 32; l++) {
			if (l == 0) entry[l] = carry;
			else {
				parse_init(entry[l].st);
				entry[l].st.p = base + l * kSeg > H ? base + l * kSeg : H;
				entry[l].last_top = entry[l].st.p;
			}
			changed[l] = true;
		}
		int it = 0;
		for (; it < 40; it++) {
			for (int l = 0; l < 32; l++) {
				if (changed[l]) {
					ex[l] = entry[l];
					cnt[l] = parse_run<false>(ex[l], base + (l + 1) * kSeg, n, lp, strategy, tabf, bytef, slowf,
					                          [](uint32_t, uint32_t, uint32_t, uint32_t) {});
				}
			}
			bool any = false;
			ParseCarry ne[32];
			for (int l = 1; l < 32; l++) ne[l] = ex[l - 1];
			changed[0] = false;
			for (int l = 1; l < 32; l++) {
				changed[l] = !carry_equal(ne[l], entry[l]);
				entry[l] = ne[l];
				any |= changed[l];
			}
			if (!any) break;
		}
		if (it > max_iters) max_iters = it;
		sum_iters += it + 1;
		++n_rounds;
		uint32_t off = total;
		for (int l = 0; l < 32; l++) {
			ParseCarry c = entry[l];
			const uint32_t o = off;
			if (syms.size() < o + cnt[l]) syms.resize(o + cnt[l]);
			uint32_t got = parse_run<true>(c, base + (l + 1) * kSeg, n, lp, strategy, tabf, bytef, slowf,
			                               [&](uint32_t k, uint32_t sym, uint32_t top, uint32_t bytes_after) {
				                               const uint32_t idx = o + k;
				                               syms[idx] = sym;
				                               if (((idx + 1) & (kBlockSyms - 1)) == 0) {
					                               const uint32_t b = (idx + 1) / kBlockSyms;
					                               blk_ptop[b - 1] = top;
					                               blk_start[b] = bytes_after;
				                               }
			                               });
			if (got != cnt[l] || !carry_equal(c, ex[l])) return 103; // final pass disagrees with the converged run
			off += cnt[l];
			if (l == 31) carry = c;
		}
		total = off;
	}
	if (getenv("B200Z_MODEL_VERBOSE")) fprintf(stderr, "parse: max propagation iterations %d, mean runs per round %.2f over %ld rounds\n", max_iters, n_rounds ? (double)sum_iters / n_rounds : 0.0, n_rounds);
	size_t nfull = total / kBlockSyms;
	const bool ended_full = !flush_then_finish && !flush_only && total > 0 && (total % kBlockSyms) == 0 && !carry.st.prevAvail;
	if (ended_full) {
		nblocks = nfull;
	} else {
		// final flush at lookahead == 0 (:750-768)
		if (carry.st.prevAvail) {
			syms.push_back(sym_lit(data[carry.st.p - 1]));
			total++;
		}
		nfull = (total - (carry.st.prevAvail ? 1 : 0)) / kBlockSyms;
		blk_ptop[nfull] = carry.last_top;
		nblocks = nfull + 1;
	}
	syms.resize(total);
	}
emit_blocks:
	Writer W;
	uint64_t bitpos = bit_base;
	std::vector<int> scratch(kTreeScratchInts + 64);
	for (size_t b = 0; b < nblocks; b++) {
		size_t s0 = b * (size_t)kBlockSyms;
		size_t s1 = s0 + kBlockSyms < syms.size() ? s0 + kBlockSyms : syms.size();
		int lit_freqs[kLiteralNum] = {0}, dist_freqs[kDistNum] = {0};
		int extra = 0;
		uint32_t blen = 0;
		for (size_t i = s0; i < s1; i++) {
			uint32_t s = syms[i];
			blen += sym_len(s);
			if (sym_dist(s) == 0) lit_freqs[s & 0xFF]++;
			else {
				int lc = lcode((int)(s & 0xFF)), dc = dcode((int)sym_dist(s) - 1);
				lit_freqs[lc]++;
				dist_freqs[dc]++;
				extra += tally_extra_bits(lc, dc);
			}
		}
		lit_freqs[256]++;
		bool last = (b + 1 == nblocks) && !flush_then_finish && !flush_only;
		int64_t storedOffset = (int64_t)blk_start[b] + abs_bias + 1 - 32768ll * (int64_t)slides_done(blk_ptop[b] + abs_bias);
		if (blk_ptop[b] >= 0xFFFFFFFEu) storedOffset = blk_ptop[b] == 0xFFFFFFFEu ? 0 : -1; // fast levels: decided by the engine
		uint8_t lit_len[kLiteralNum], dist_len[kDistNum];
		uint16_t lit_codes[kLiteralNum], dist_codes[kDistNum];
		uint32_t hdr[192];
		std::memset(hdr, 0, sizeof(hdr));
		BlockPlan plan;
		plan_block(lit_freqs, dist_freqs, extra, storedOffset >= 0, (int)blen, last, lit_len, lit_codes, dist_len,
		           dist_codes, hdr, scratch.data(), plan);
		if (plan.type == 0) {
			W.put(bitpos, hdr[0], 3);
			bitpos += 3;
			bitpos = (bitpos + 7) & ~7ull;
			W.put(bitpos, blen & 0xFFFF, 16);
			W.put(bitpos + 16, (~blen) & 0xFFFF, 16);
			bitpos += 32;
			for (uint32_t i = 0; i < blen; i++) {
				W.put(bitpos, data[blk_start[b] + i], 8);
				bitpos += 8;
			}
		} else {
			for (uint32_t i = 0; i < plan.hdr_bits; i += 32) {
				int nb = plan.hdr_bits - i < 32 ? (int)(plan.hdr_bits - i) : 32;
				W.put(bitpos + i, hdr[i >> 5] & (nb == 32 ? 0xFFFFFFFFu : ((1u << nb) - 1)), nb);
			}
			bitpos += plan.hdr_bits;
			uint64_t body0 = bitpos;
			for (size_t i = s0; i < s1; i++) {
				uint64_t bits;
				int nb;
				encode_symbol(syms[i], lit_codes, lit_len, dist_codes, dist_len, bits, nb);
				W.put(bitpos, bits, nb);
				bitpos += nb;
			}
			W.put(bitpos, lit_codes[256], lit_len[256]);
			bitpos += lit_len[256];
			if (bitpos - body0 != plan.body_bits) return 101; // planner and emitter disagree
		}
	}
	if (flush_then_finish || flush_only) {
		// Deflater.Deflate FLUSHING_STATE (:486-504) then Finish: an empty final static block
		int neededbits = 8 + (int)((0 - bitpos) & 7);
		while (neededbits > 0) {
			W.put(bitpos, 2, 10);
			bitpos += 10;
			neededbits -= 10;
		}
		if (flush_then_finish) {
			W.put(bitpos, 3, 10);
			bitpos += 10;
		}
	}
	*outbits = bitpos;
	uint64_t nbytes = (bitpos + 7) >> 3;
	if (nbytes > cap) return 102;
	W.w.resize((nbytes + 3) / 4 + 1, 0);
	std::memcpy(out, W.w.data(), nbytes);
	*outlen = nbytes;
	return 0;
}
