// b200z_inflate_par.cuh -- the block-parallel inflate pipeline (included by b200z_inflate.cu).
//
// The reference's Inflater (Zip/Compression/Inflater.cs:429-552) walks a stream bit by bit; across a block boundary it
// carries nothing but the bit position and the window (= the output so far).  That is the parallelism used here:
//
//   k_find / k_find3   every bit offset of every stream is tested for "a dynamic block header could start here" (BFINAL = 0,
//                      BTYPE = 2, HLIT / HDIST in range, a complete code-length code, code lengths that decode to exactly
//                      HLIT + HDIST entries with an end-of-block code and complete literal and distance codes).  The first
//                      survivor of every 8192-bit window of a stream is a CANDIDATE.  Candidates are hints, nothing more.
//   k_seglist          the stream starts and the candidates become the SEGMENT list.
//   k_dec1             persistent CTAs take segments off the list and decode them without writing output: block headers
//                      (InflaterDynHeader.cs:42-120), code tables (InflaterHuffmanTree.cs:87-169) and ROUNDS of 128 lanes x
//                      512 bits -- every lane decodes its sub-chunk speculatively, exit -> entry hand-off until stable, the
//                      same scheme as the serial kernel, four warps wide.  A segment ends when the position it has reached
//                      at a block boundary is itself a candidate (someone else decodes on from there: the two decoders are
//                      the same deterministic function of the bit position, so the hand-over is exact), at the final block,
//                      at an error or at the end of the input.  Per round it records every lane's entry position and the
//                      prefix sums of the bytes and back-references the lanes produce.
//   k_chain            one thread per stream follows the segments from the stream start (join -> the candidate's segment
//                      -> ...), gives every segment on the chain its output position, and derives what Inflater reports:
//                      status, TotalOut, RemainingInput (trap T14), the restart and resume points.
//   k_dec2             one CTA per recorded batch of rounds: the final decode pass, every lane from its recorded entry with
//                      its recorded output position -- literals straight into the output buffer, back-references as
//                      (position, length, distance) records in stream order.
//   k_resolve          one CTA per stream walks the output in 16 KiB tiles: every byte of a back-reference points at its
//                      source byte (OutputWindow.Repeat's rule, Streams/OutputWindow.cs:63-92: byte k of a copy comes from
//                      source byte k mod distance), sources in front of the tile are final and read directly, pointers inside
//                      the tile are resolved by pointer jumping in shared memory, the tile is written back.
//
// Anything that does not fit the pipeline's fixed pools (pathological streams of thousands of tiny blocks, outputs beyond
// 4 GiB) is flagged and decoded by the serial kernel k_inflate afterwards; results are identical by construction, the
// serial kernel is the reference point the parallel one is tested against.
#pragma once

namespace b200z {

constexpr int kFWShift = 13; // candidate windows of 8192 bits
constexpr uint32_t kFWMask = (1u << kFWShift) - 1u;
constexpr uint32_t kNoCand = 0xFFFFFFFFu;
constexpr int kP1Threads = 128;                              // lanes of a round
constexpr int kP1RoundWords = kP1Threads * kSubBits / 32;   // 2048 words of input per round
constexpr int kP1InWords = kP1RoundWords + 8;
constexpr int kP1InSlots = kP1InWords + kP1InWords / 16 + 1;
constexpr int kRoundBatch = 4;                               // rounds are allocated four at a time, a batch never mixes blocks
constexpr int kFindTileWords = 2048;
constexpr int kResTile = 16384;                              // k_resolve: bytes per tile
constexpr int kResThreads = 1024;

enum { SEG_JOIN = 0, SEG_FINAL = 1, SEG_STOP = 2, SEG_POOL = 3 };
enum { RND_NONE = 0, RND_HUFF = 1, RND_STORED = 2 };

struct FTile { // k_find: 2048 words of one stream
	uint32_t stream, word0, nwords, pad;
};

struct __align__(16) PSeg {
	uint64_t start_bit, end_bit, rs_bit;
	uint64_t body_bit;          // where the symbols of the block at rs_bit start (rs_bit: a stored block or an unfinished header)
	uint64_t out_bytes, rs_out; // relative to the segment's first output byte
	uint64_t out_base;          // k_chain: output position of the segment
	uint32_t stream, n_match, match_base;
	int32_t end_kind, status;
	uint32_t valid;
};

struct __align__(16) PRound {
	uint32_t seg, kind, hdr, w0;            // hdr: index of the block's PBlockHdr; w0: first staged word (stored: source byte offset)
	uint32_t r0, end_rel, lastlane, nbytes; // stored: nbytes = LEN
	uint64_t out_rel;                       // relative to the segment
	uint32_t match_rel, pad;
	uint32_t entry[kP1Threads];
	uint32_t opre[kP1Threads]; // exclusive prefix sums over the lanes: output bytes / back-references
	uint32_t mpre[kP1Threads];
};

struct __align__(16) PBlockHdr { // a block's code tables as k_dec1 built them, for k_dec2
	InfShared tab;
};

struct PCounters {
	uint32_t fs_count, nseg, seg_next, round_top, hdr_top;
	uint32_t n_rounds, n_passes, n_blocks; // statistics (b200z_plan_get_stats)
};

// ---------------------------------------------------------------------------------------------------------
// finder
// ---------------------------------------------------------------------------------------------------------
// Stages 1 and 2.  32 bit offsets at a time: the fixed header fields as bit-parallel masks over funnel-shifted words; the
// positions that pass (11 %) are compacted per warp so that every lane has one to test, then the Kraft sum of the
// code-length code (a complete code: sum of 2^(7-len) = 128) through a table of four lengths at a time.
__global__ void __launch_bounds__(256)
    k_find(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
           const FTile *__restrict__ tiles, const uint32_t *__restrict__ start_bit, const int64_t *__restrict__ skip_bit,
           const int32_t *__restrict__ pre, unsigned long long *__restrict__ fs_list, PCounters *__restrict__ ctr, uint32_t fs_cap) {
	__shared__ uint8_t lut[4096];
	__shared__ uint32_t sw[kFindTileWords + 4];
	__shared__ uint16_t queue[8][1024];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int i = threadIdx.x; i < 4096; i += 256) {
		uint32_t s = 0;
		for (int j = 0; j < 4; j++) {
			const uint32_t l = ((uint32_t)i >> (3 * j)) & 7u;
			if (l) s += 128u >> l;
		}
		lut[i] = (uint8_t)(s > 255u ? 255u : s);
	}
	const FTile t = tiles[blockIdx.x];
	if (pre && pre[t.stream] != B200Z_OK) return;
	const uint32_t *gwords = reinterpret_cast<const uint32_t *>(in + in_off[t.stream]);
	const uint32_t nbytes = (uint32_t)in_len[t.stream];
	const uint32_t nwords = (nbytes + 3) >> 2;
	uint64_t sb = start_bit ? start_bit[t.stream] : 0u;
	// a stream entered in mid-block (b200z_inflate_plan_set_resume): its chain jumps from the header copy to skip_bit, so
	// nothing in front of that is a block it could join
	if (skip_bit && (uint64_t)skip_bit[t.stream] > sb) sb = (uint64_t)skip_bit[t.stream];
	const uint64_t total_bits = 8ull * nbytes;
	for (uint32_t i = threadIdx.x; i < t.nwords + 4; i += 256) sw[i] = ld_stream_word(gwords, t.word0 + i, nwords, nbytes);
	__syncthreads();
	uint16_t *q = queue[warp];
	for (uint32_t base = (uint32_t)warp * 32u; base < t.nwords; base += 256u) {
		const uint32_t k = base + (uint32_t)lane;
		uint32_t mask = 0;
		if (k < t.nwords) {
			const uint32_t w0 = sw[k], w1 = sw[k + 1];
#define B200Z_S(kk) __funnelshift_r(w0, w1, kk)
			mask = ~w0 & ~B200Z_S(1) & B200Z_S(2);                           // BFINAL = 0, BTYPE = 2 (bits 1, 2 = 0, 1)
			mask &= ~(B200Z_S(4) & B200Z_S(5) & B200Z_S(6) & B200Z_S(7));    // HLIT <= 29
			mask &= ~(B200Z_S(9) & B200Z_S(10) & B200Z_S(11) & B200Z_S(12)); // HDIST <= 29
#undef B200Z_S
			const uint64_t wbit = 32ull * (t.word0 + k);
			if (wbit + 32 <= sb) mask = 0;
			else if (wbit <= sb) { // nothing in front of the stream's first block header, and not that header itself (segment 0 has it)
				const uint32_t cut = (uint32_t)(sb - wbit) + 1;
				mask = cut >= 32 ? 0u : (mask >> cut) << cut;
			}
		}
		const uint32_t cnt = (uint32_t)__popc(mask);
		uint32_t incl = cnt;
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += v;
		}
		const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
		{
			uint32_t pos = incl - cnt, m = mask;
			while (m) {
				const uint32_t o = (uint32_t)__ffs((int)m) - 1u;
				m &= m - 1u;
				q[pos++] = (uint16_t)(((uint32_t)lane << 5) | o);
			}
		}
		__syncwarp();
		for (uint32_t e = (uint32_t)lane; e < total; e += 32u) {
			const uint32_t ent = q[e];
			const uint32_t wl = base + (ent >> 5), o = ent & 31u;
			const uint32_t sh = o + 13u; // HCLEN and the code-length code's lengths: 4 + 57 bits from here
			const bool lowh = sh < 32u;
			const uint32_t a = lowh ? sw[wl] : sw[wl + 1], b = lowh ? sw[wl + 1] : sw[wl + 2], c = lowh ? sw[wl + 2] : sw[wl + 3];
			uint32_t v0 = __funnelshift_r(a, b, sh), v1 = __funnelshift_r(b, c, sh);
			const uint32_t nmeta = (v0 & 15u) + 4u;
			const uint32_t nb = 4u + 3u * nmeta; // 16 .. 61 bits in use
			if (nb >= 32u) v1 &= (1u << (nb - 32u)) - 1u;
			else {
				v1 = 0;
				v0 &= (1u << nb) - 1u;
			}
			const uint32_t sum = (uint32_t)lut[(v0 >> 4) & 4095u] + lut[(v0 >> 16) & 4095u] + lut[__funnelshift_r(v0, v1, 28) & 4095u] +
			                     lut[(v1 >> 8) & 4095u] + lut[(v1 >> 20) & 4095u];
			if (sum != 128u) continue;
			const uint64_t pos = 32ull * (t.word0 + wl) + o;
			if (pos + 17 + 3 * nmeta > total_bits) continue;
			const uint32_t idx = atomicAdd(&ctr->fs_count, 1u);
			if (idx < fs_cap) fs_list[idx] = ((unsigned long long)t.stream << 40) | pos;
		}
		__syncwarp();
	}
}

// Stage 3, one thread per survivor: the code lengths themselves (InflaterDynHeader.cs:62-117's rules) and the two codes
// they describe.  What passes is entered as its window's candidate (the lowest position wins).
__global__ void __launch_bounds__(128)
    k_find3(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
            const unsigned long long *__restrict__ fs_list, const PCounters *__restrict__ ctr, uint32_t fs_cap,
            const uint32_t *__restrict__ win_base, uint32_t *__restrict__ cand) {
	__shared__ uint8_t s_tab[128 * 128];
	uint32_t count = ctr->fs_count;
	if (count > fs_cap) count = fs_cap;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
		const unsigned long long e = fs_list[i];
		const uint32_t stream = (uint32_t)(e >> 40);
		const uint64_t pos = e & ((1ull << 40) - 1ull);
		BitReader br = BitReader::at(reinterpret_cast<const uint32_t *>(in + in_off[stream]), (uint32_t)in_len[stream], pos);
		br.get(3);
		const int nlit = (int)br.get(5) + 257, ndist = (int)br.get(5) + 1, nmeta = (int)br.get(4) + 4;
		// the code-length code's lengths, 3 bits each, kept in one word per ten symbols
		uint32_t mlo = 0, mhi = 0; // symbol s: bits 3 (s % 10) of (s < 10 ? mlo : mhi)
		for (int k = 0; k < nmeta; k++) {
			const uint32_t sym = c_meta_order[k], v = br.get(3);
			if (sym < 10) mlo |= v << (3 * sym);
			else mhi |= v << (3 * (sym - 10));
		}
		// 7-bit decode table of the code-length code in shared memory: sym << 3 | len; column tid of a [128][128] byte array
		uint8_t *tab = s_tab + threadIdx.x;
		for (int k = 0; k < 128; k++) tab[k * 128] = 0;
		{
			uint32_t cnt[8], nxt[8];
			for (int L = 0; L < 8; L++) cnt[L] = 0;
			for (int s = 0; s < 19; s++) cnt[((s < 10 ? mlo >> (3 * s) : mhi >> (3 * (s - 10))) & 7u)]++;
			cnt[0] = 0;
			uint32_t code = 0;
			for (int L = 1; L <= 7; L++) {
				nxt[L] = code;
				code = (code + cnt[L]) << 1;
			}
			for (int s = 0; s < 19; s++) {
				const uint32_t L = (s < 10 ? mlo >> (3 * s) : mhi >> (3 * (s - 10))) & 7u;
				if (!L) continue;
				const uint32_t c = nxt[L]++;
				const uint32_t rev = __brev(c) >> (32 - L);
				for (uint32_t k = rev; k < 128u; k += (1u << L)) tab[k * 128] = (uint8_t)((s << 3) | L);
			}
		}
		const int total = nlit + ndist;
		int idx = 0, prev = 0, nd = 0, eob_len = 0;
		uint32_t kl = 0, kd = 0;
		bool ok = true;
		while (ok && idx < total) {
			br.refill();
			const uint32_t te = tab[br.peek(7) * 128];
			if (!te) { ok = false; break; }
			br.drop((int)(te & 7u));
			const int sym = (int)(te >> 3);
			int rep = 1, val = sym;
			if (sym == 16) {
				if (idx == 0) { ok = false; break; }
				val = prev;
				rep = 3 + (int)br.get(2);
			} else if (sym == 17) {
				val = 0;
				rep = 3 + (int)br.get(3);
			} else if (sym == 18) {
				val = 0;
				rep = 11 + (int)br.get(7);
			}
			if (idx + rep > total) { ok = false; break; }
			{
				// `rep` entries of length `val` from index idx on: how many are literal/length codes, how many distance codes
				const int nl = idx >= nlit ? 0 : (nlit - idx < rep ? nlit - idx : rep), ndc = rep - nl;
				if (idx <= 256 && 256 < idx + rep) eob_len = val;
				if (val) {
					kl += (uint32_t)nl * (32768u >> val);
					kd += (uint32_t)ndc * (32768u >> val);
					nd += ndc;
				}
				idx += rep;
			}
			prev = val;
			if (br.overrun()) ok = false;
		}
		if (!ok || br.overrun() || eob_len == 0 || kl != 32768u || !(kd == 32768u || nd <= 1)) continue;
		atomicMin(&cand[win_base[stream] + (uint32_t)(pos >> kFWShift)], (uint32_t)pos & kFWMask);
	}
}

// the segment list: slots 0 .. n-1 are the stream starts, slot n + g is window g's candidate
__global__ void k_seglist(int n, uint32_t nwin_total, const uint32_t *__restrict__ win_base, const uint32_t *__restrict__ win_stream,
                          const uint32_t *__restrict__ cand, const uint32_t *__restrict__ start_bit, const int32_t *__restrict__ pre,
                          PSeg *__restrict__ segs, uint32_t *__restrict__ seg_list, PCounters *__restrict__ ctr) {
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= (uint32_t)n + nwin_total) return;
	uint32_t stream;
	uint64_t sbit;
	if (slot < (uint32_t)n) {
		stream = slot;
		if (pre && pre[stream] != B200Z_OK) return;
		sbit = start_bit ? start_bit[stream] : 0u;
	} else {
		const uint32_t g = slot - (uint32_t)n;
		const uint32_t c = cand[g];
		if (c == kNoCand) return;
		stream = win_stream[g];
		sbit = ((uint64_t)(g - win_base[stream]) << kFWShift) + c;
	}
	PSeg &s = segs[slot];
	s.stream = stream;
	s.start_bit = sbit;
	s.valid = 0;
	s.end_kind = SEG_STOP;
	s.status = B200Z_E_INTERNAL;
	seg_list[atomicAdd(&ctr->nseg, 1u)] = slot;
}

// ---------------------------------------------------------------------------------------------------------
// code tables, built by the whole CTA (the same tables build_table() makes serially)
// ---------------------------------------------------------------------------------------------------------
struct TabScratch {
	uint32_t cnt[2][16], nxt[2][16], run[2][16];
	int err;
};

// lens[0 .. nlit) literal/length code lengths, lens[nlit .. nlit + ndist) distance code lengths.  All threads of the CTA
// (>= 64) call it; returns 0 or a detail code, the same for every thread.
__device__ int build_tables_cta(InfShared &sh, TabScratch &ts, int nlit, int ndist) {
	const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, warp = tid >> 5;
	for (int i = tid; i < (1 << kLitRoot); i += nthr) sh.lit[i] = 0;
	for (int i = tid; i < (1 << kDistRoot); i += nthr) sh.dist[i] = 0;
	if (tid < 32) {
		ts.cnt[tid >> 4][tid & 15] = 0;
		ts.run[tid >> 4][tid & 15] = 0;
	}
	if (tid == 0) ts.err = 0;
	__syncthreads();
	for (int s = tid; s < nlit; s += nthr) {
		const int L = sh.lens[s];
		if (L) atomicAdd(&ts.cnt[0][L], 1u);
	}
	for (int s = tid; s < ndist; s += nthr) {
		const int L = sh.lens[nlit + s];
		if (L) atomicAdd(&ts.cnt[1][L], 1u);
	}
	__syncthreads();
	if (tid < 2) {
		const int d = canon_setup(ts.cnt[tid], ts.nxt[tid], tid ? &sh.dist_c : &sh.lit_c, tid ? kDistRoot : kLitRoot);
		if (d) ts.err = d;
	}
	__syncthreads();
	const int err = ts.err;
	if (err) return err;
	if (warp < 2) {
		// warp 0: literal/length symbols in order, warp 1: distance symbols; the canonical code of symbol s is
		// next[L] + (number of earlier symbols of the same length)
		const int k = warp, n = k ? ndist : nlit, R = k ? kDistRoot : kLitRoot;
		const uint8_t *lens = sh.lens + (k ? nlit : 0);
		uint32_t *tab = k ? sh.dist : sh.lit;
		uint16_t *sorted = k ? sh.dist_sorted : sh.lit_sorted;
		const Canon &cn = k ? sh.dist_c : sh.lit_c;
		const uint32_t size = 1u << R;
		for (int base = 0; base < n; base += 32) {
			const int s = base + lane;
			const int L = s < n ? lens[s] : 0;
			const uint32_t m = __match_any_sync(0xffffffffu, L);
			const uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1u));
			const uint32_t r0 = ts.run[k][L];
			__syncwarp();
			if (L && lane == __ffs((int)m) - 1) ts.run[k][L] = r0 + (uint32_t)__popc(m);
			__syncwarp();
			if (L) {
				const uint32_t c = ts.nxt[k][L] + r0 + rank;
				const uint32_t rev = __brev(c) >> (32 - L);
				if (L <= R) {
					const uint32_t e = k == 0 ? litlen_entry((uint32_t)s, (uint32_t)L) : dist_entry((uint32_t)s, (uint32_t)L);
					for (uint32_t i = rev; i < size; i += (1u << L)) tab[i] = e;
				} else {
					sorted[cn.offs[L] + (c - cn.first[L])] = (uint16_t)s;
					tab[rev & (size - 1u)] = mk_entry(0, K_LONG, 0, 0);
				}
			}
		}
	}
	__syncthreads();
	return 0;
}

// ---------------------------------------------------------------------------------------------------------
// span decode without per-lane caps.  MODE 0 counts; MODE 1 stores literals at out[o0 + o] and back-references at
// ml[nm] (output positions relative to the stream).
// ---------------------------------------------------------------------------------------------------------
// One symbol per call, the common cases without a branch: the lanes of a warp step together, and with 32 of them some
// lane always holds a literal and some lane a back-reference, so both paths would be paid for anyway.  Every lane peeks
// twice (the literal/length code, and what follows its extra bits -- the distance code if it was a length) and selects.
// Codes longer than the root tables, end of block and the error cases leave through rare branches.

// A lane's decode state: the bit position and, in registers, the next 33..64 bits of the stream from there (refilled 32 bits
// at a time from the staged words), so that a literal costs one table lookup and a few shifts -- no shared-memory round
// trip for the bits themselves.
struct SpanB {
	uint64_t bb;   // stream bits from `pos` on, least significant first
	uint32_t nb;   // how many of them are valid
	uint32_t widx; // next staged word to take
	uint32_t pos, o, nm, fl, det;
};

__device__ __forceinline__ void span_begin(SpanB &s, const uint32_t *words, uint32_t pos) {
	const uint32_t i = pos >> 5, sh = pos & 31u;
	const uint64_t two = (uint64_t)words[in_slot(i)] | ((uint64_t)words[in_slot(i + 1)] << 32);
	s.bb = two >> sh;
	s.nb = 64u - sh;
	s.widx = i + 2;
	s.pos = pos;
	s.o = 0;
	s.nm = 0;
	s.fl = 0;
	s.det = 0;
}
__device__ __forceinline__ void span_refill(SpanB &s, const uint32_t *words) { // afterwards at least 33 bits are valid
	if (s.nb <= 32u) {
		s.bb |= (uint64_t)words[in_slot(s.widx)] << s.nb;
		s.nb += 32u;
		++s.widx;
	}
}
__device__ __forceinline__ void span_drop(SpanB &s, uint32_t n) {
	s.bb >>= n;
	s.nb -= n;
	s.pos += n;
}

// One symbol.  MODE 0 counts; MODE 1 stores literals at out[o0 + o] and back-references at ml[nm] (output positions relative
// to the stream).  A symbol that needs bits past the end of the input is not consumed (pos stays at its first bit).
template <int MODE>
__device__ __forceinline__ bool span_step2(const InfShared &sh, const uint32_t *words, SpanB &s, uint32_t limit, uint32_t end_rel,
                                           uint8_t *out, uint64_t o0, MatchTok *ml) {
	const uint32_t spos = s.pos;
	if (spos >= limit) return false;
	span_refill(s, words);
	const uint32_t v = (uint32_t)s.bb;
	uint32_t e = sh.lit[v & ((1u << kLitRoot) - 1u)];
	uint32_t k = (e >> 4) & 15u;
	if (k == K_LIT) {
		const uint32_t nb = e & 15u;
		if (spos + nb > end_rel) { s.fl |= F_OVERRUN; return false; }
		if (MODE) out[o0 + s.o] = (uint8_t)(e >> 16);
		++s.o;
		span_drop(s, nb);
		return true;
	}
	if (k == K_LONG) {
		e = long_code(v, sh.lit_sorted, sh.lit_c, kLitRoot, 0);
		k = (e >> 4) & 15u;
		if (k == K_LIT) {
			const uint32_t nb = e & 15u;
			if (spos + nb > end_rel) { s.fl |= F_OVERRUN; return false; }
			if (MODE) out[o0 + s.o] = (uint8_t)(e >> 16);
			++s.o;
			span_drop(s, nb);
			return true;
		}
	}
	const uint32_t nb = e & 15u;
	if (k == K_LEN) {
		// length code (<= 15 bits) + extra (<= 5) are in the buffer; the distance code + extra (<= 28) after a refill
		const uint32_t xb = (e >> 8) & 15u;
		const uint32_t len = (e >> 16) + ((v >> nb) & ((1u << xb) - 1u));
		const uint32_t pos1 = spos + nb + xb;
		uint64_t bb = s.bb >> (nb + xb);
		uint32_t have = s.nb - (nb + xb), widx = s.widx;
		if (have <= 32u) {
			bb |= (uint64_t)words[in_slot(widx)] << have;
			have += 32u;
			++widx;
		}
		const uint32_t v2 = (uint32_t)bb;
		uint32_t de = sh.dist[v2 & ((1u << kDistRoot) - 1u)];
		if (((de >> 4) & 15u) == K_LONG) de = long_code(v2, sh.dist_sorted, sh.dist_c, kDistRoot, 1);
		const uint32_t dk = (de >> 4) & 15u, dnb = de & 15u;
		if (dk != K_DIST) {
			// Invalid codes near the end of the input, as the reference classifies them (InflaterHuffmanTree.GetSymbol :181-235):
			// a table entry without a code is diagnosed as soon as 9 bits can be peeked; a code for an illegal symbol (286, 287,
			// distance 30, 31) once its own bits are there; with fewer bits the decoder waits for more input.
			if (pos1 + (dk == K_ILLEGAL ? dnb : 9u) > end_rel) s.fl |= F_OVERRUN;
			else { s.fl |= F_ERR; s.det = dk == K_ILLEGAL ? D_REP_DIST : D_CODELEN0; }
			return false;
		}
		const uint32_t dxb = (de >> 8) & 15u;
		const uint32_t dist = (de >> 16) + ((v2 >> dnb) & ((1u << dxb) - 1u));
		const uint32_t npos = pos1 + dnb + dxb;
		if (npos > end_rel) { s.fl |= F_OVERRUN; return false; }
		if (MODE) {
			MatchTok t;
			t.out_pos = (uint32_t)(o0 + s.o);
			t.len = (uint16_t)len;
			t.dist = (uint16_t)(dist & 0xFFFFu); // 32768 fits
			ml[s.nm] = t;
		}
		++s.nm;
		s.o += len;
		s.bb = bb >> (dnb + dxb);
		s.nb = have - (dnb + dxb);
		s.widx = widx;
		s.pos = npos;
		return true;
	}
	if (k == K_EOB) {
		if (spos + nb > end_rel) s.fl |= F_OVERRUN;
		else { s.fl |= F_EOB; s.pos = spos + nb; }
		return false;
	}
	if (spos + (k == K_ILLEGAL ? nb : 9u) > end_rel) s.fl |= F_OVERRUN;
	else { s.fl |= F_ERR; s.det = k == K_ILLEGAL ? D_REP_LEN : D_CODELEN0; }
	return false;
}

// ---------------------------------------------------------------------------------------------------------
// k_dec1: counted decode of segments
// ---------------------------------------------------------------------------------------------------------
struct __align__(16) Dec1Shared {
	InfShared sh;
	TabScratch ts;
	uint32_t in[kP1InSlots];
	uint32_t exitp[kP1Threads], flags[kP1Threads], dets[kP1Threads];
	uint32_t wsum_o[4], wsum_m[4];
	// header results (thread 0 -> all)
	int h_st, h_detail, h_btype, h_last, h_nlit, h_ndist;
	unsigned long long h_bitpos;
	unsigned long long h_body; // thread 0 only: where the current block's symbols start (its header bit if it has none)
	uint32_t h_stored_len;
	uint32_t q_idx, a_base;
	int stop[2], front[2];
	uint32_t nlive[2];
};

__global__ void __launch_bounds__(kP1Threads, 10) // 48 registers: ten CTAs per SM (the header parse would take 64)
    k_dec1(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len, PSeg *__restrict__ segs,
           const uint32_t *__restrict__ seg_list, PCounters *__restrict__ ctr, const uint32_t *__restrict__ win_base,
           const uint32_t *__restrict__ cand, PRound *__restrict__ rounds, uint32_t round_cap, PBlockHdr *__restrict__ hdrs,
           uint32_t hdr_cap, const int64_t *__restrict__ skip_bit) {
	extern __shared__ __align__(16) uint8_t smem_raw[];
	Dec1Shared &S = *reinterpret_cast<Dec1Shared *>(smem_raw);
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint32_t nseg = ctr->nseg;
	for (;;) {
		__syncthreads();
		if (tid == 0) S.q_idx = atomicAdd(&ctr->seg_next, 1u);
		__syncthreads();
		const uint32_t qi = S.q_idx;
		if (qi >= nseg) break;
		const uint32_t slot = seg_list[qi];
		PSeg &seg = segs[slot];
		const uint32_t stream = seg.stream;
		const uint32_t *gwords = reinterpret_cast<const uint32_t *>(in + in_off[stream]);
		const uint32_t nbytes = (uint32_t)in_len[stream];
		const uint32_t nwords = (nbytes + 3) >> 2;
		const uint64_t total_bits = 8ull * nbytes;
		const uint32_t wb = win_base[stream], nwin = win_base[stream + 1] - wb;

		// uniform across the CTA
		uint64_t bitpos = seg.start_bit, opos = 0, rs_bit = bitpos, rs_out = 0;
		uint32_t nm_total = 0;
		int st = B200Z_OK, detail = 0, end_kind = SEG_STOP;
		bool last = false;
		uint32_t blocks_done = 0;
		for (;;) { // blocks
			if (last) { // Inflater.cs:443-449: raw mode stops right behind the final block
				end_kind = SEG_FINAL;
				break;
			}
			if (blocks_done) { // a block boundary that is a candidate: its segment decodes on from here
				const uint64_t w = bitpos >> kFWShift;
				if (w < nwin && cand[wb + (uint32_t)w] == ((uint32_t)bitpos & kFWMask)) {
					end_kind = SEG_JOIN;
					break;
				}
			}
			rs_bit = bitpos;
			rs_out = opos;
			// ---- block header (thread 0) -----------------------------------------------------------------------
			if (tid == 0) {
				BitReader br = BitReader::at(gwords, nbytes, bitpos);
				BlockHeader h = read_block_header(br, S.sh);
				S.h_body = (h.status == B200Z_OK && (h.btype == 1 || h.btype == 2)) ? br.consumed : bitpos;
				// the stream-start segment (slot == stream) of a stream entered in mid-block: the header is a copy
				if (!blocks_done && slot == stream && skip_bit) enter_mid_block(h, br, (uint64_t)skip_bit[stream]);
				S.h_st = h.status;
				S.h_detail = h.detail;
				S.h_btype = h.btype;
				S.h_last = h.last;
				S.h_nlit = h.nlit;
				S.h_ndist = h.ndist;
				S.h_bitpos = br.consumed;
				S.h_stored_len = h.stored_len;
			}
			__syncthreads();
			st = S.h_st;
			detail = S.h_detail;
			const int btype = S.h_btype;
			bitpos = S.h_bitpos;
			if (st != B200Z_OK) break;
			last = S.h_last != 0;
			uint32_t batch_base = 0, batch_used = kRoundBatch; // rounds of this block
			if (btype == 0) {
				// ---- stored block: recorded, copied by k_dec2 (OutputWindow.CopyStored :100-122) -----------------------
				const uint32_t stored_len = S.h_stored_len;
				const uint64_t ipos = bitpos >> 3;
				const uint64_t avail = ipos <= nbytes ? nbytes - ipos : 0;
				if (stored_len > avail) {
					st = B200Z_E_NEED_INPUT;
					break;
				}
				if (tid == 0) S.a_base = atomicAdd(&ctr->round_top, (uint32_t)kRoundBatch);
				__syncthreads();
				batch_base = S.a_base;
				if (batch_base + kRoundBatch > round_cap) {
					end_kind = SEG_POOL;
					break;
				}
				if (tid == 0) {
					PRound &r = rounds[batch_base];
					r.seg = slot;
					r.kind = RND_STORED;
					r.hdr = 0;
					r.w0 = (uint32_t)ipos;
					r.nbytes = stored_len;
					r.out_rel = opos;
					r.match_rel = nm_total;
					for (int k = 1; k < kRoundBatch; k++) rounds[batch_base + k].kind = RND_NONE;
				}
				opos += stored_len;
				bitpos = 8ull * (ipos + stored_len);
				++blocks_done;
				continue;
			}
			// ---- Huffman block: code tables ---------------------------------------------------------------------
			int nlit = S.h_nlit, ndist = S.h_ndist;
			if (btype == 1) {
				__syncthreads();
				static_lens(S.sh.lens, tid, (int)blockDim.x);
				nlit = 288;
				ndist = 32;
				__syncthreads();
			}
			{
				const int d = build_tables_cta(S.sh, S.ts, nlit, ndist);
				if (d) {
					st = B200Z_E_DATA;
					detail = d;
					break;
				}
			}
			if (tid == 0) {
				S.a_base = atomicAdd(&ctr->hdr_top, 1u);
				atomicAdd(&ctr->n_blocks, 1u);
			}
			__syncthreads();
			const uint32_t hdr_idx = S.a_base;
			if (hdr_idx >= hdr_cap) {
				end_kind = SEG_POOL;
				break;
			}
			{
				const uint4 *src = reinterpret_cast<const uint4 *>(&S.sh);
				uint4 *dstv = reinterpret_cast<uint4 *>(&hdrs[hdr_idx].tab);
				for (int i = tid; i < (int)(sizeof(InfShared) / 16); i += kP1Threads) dstv[i] = src[i];
			}
			// ---- rounds -------------------------------------------------------------------------------------------
			bool in_block = true;
			while (in_block) {
				__syncthreads();
				if (tid == 0) {
					S.stop[0] = S.stop[1] = kP1Threads - 1;
					S.front[0] = S.front[1] = kP1Threads;
					S.nlive[0] = S.nlive[1] = 0;
				}
				const uint32_t w0 = (uint32_t)(bitpos >> 5);
				stage_words(S.in, gwords, w0, kP1InWords, nwords, nbytes, tid, (int)blockDim.x);
				__syncthreads();
				const uint32_t *words = S.in;
				const uint32_t r0 = (uint32_t)(bitpos & 31);
				const uint64_t remain = total_bits - ((uint64_t)w0 << 5);
				const uint32_t end_rel = remain > 0x7FFFFFFFull ? 0x7FFFFFFFu : (uint32_t)remain;
				const uint32_t limit = r0 + (uint32_t)(tid + 1) * kSubBits;
				uint32_t entry = r0 + (uint32_t)tid * kSubBits;
				uint32_t obytes = 0, nmatch = 0, flags = 0;
				bool need = true, dead = false;
				uint32_t passes = 0, nlive = kP1Threads, runs = 0;
				int lastlane = kP1Threads - 1, front = 0;
				// Lane 0 starts at the true position, the others at a guess; every pass a lane whose entry moved (to the
				// previous lane's exit) decodes again.  The first lane that stops the block (end of block, error, end of
				// input) kills the lanes behind it at once: S.stop[pass parity] collects the lowest such lane.
				// Codes that re-synchronise (text: within ~120 bits) settle in three or four passes.  Codes that do not (nearly
				// flat ones: incompressible data in Huffman blocks) would have every lane behind the exact ones decode garbage
				// again in every pass; so a lane decodes on a guess twice at most, and after that, while more than 16 lanes
				// still wait, only the lowest waiting lane -- whose entry is exact, all lanes in front of it being settled --
				// decodes: the round degrades to one serial decoder instead of 128 useless ones.
				for (int it = 0; it < 2 * kP1Threads + 8; it++) {
					++passes;
					const bool run = need && !dead && (runs < 2u || nlive <= 16u || tid == front);
					SpanB sp;
					bool act = run;
					if (run) span_begin(sp, words, entry);
					while (__any_sync(0xffffffffu, act)) {
						if (act) act = span_step2<0>(S.sh, words, sp, limit, end_rel, nullptr, 0, nullptr);
						__syncwarp();
					}
					if (run) {
						obytes = sp.o;
						nmatch = sp.nm;
						flags = sp.fl;
						S.exitp[tid] = sp.pos;
						S.flags[tid] = sp.fl;
						S.dets[tid] = sp.det;
						need = false;
						++runs;
					} else if (need && dead) {
						flags = (uint32_t)F_DEAD;
						S.flags[tid] = (uint32_t)F_DEAD;
						need = false;
					}
					if (flags & (F_EOB | F_ERR | F_OVERRUN)) atomicMin(&S.stop[it & 1], tid);
					if (tid == 0) S.stop[(it + 1) & 1] = kP1Threads - 1; // (last read before the previous pass's second barrier)
					__syncthreads();
					lastlane = S.stop[it & 1];
					const bool nd = tid > lastlane;
					if (nd != dead) {
						need = true;
						runs = 0; // (back from behind a stop that went away: its guesses count afresh)
					}
					dead = nd;
					if (tid > 0 && !nd) { // (a dead lane's entry does not matter; it is taken afresh should the lane come back)
						const uint32_t pe = S.exitp[tid - 1];
						if (pe != entry) {
							entry = pe;
							need = true;
						}
					}
					if (tid == 0) { // (last read behind the previous pass's second barrier, in front of this pass's first)
						S.front[(it + 1) & 1] = kP1Threads;
						S.nlive[(it + 1) & 1] = 0;
					}
					if (need && !dead) {
						atomicMin(&S.front[it & 1], tid);
						atomicAdd(&S.nlive[it & 1], 1u);
					}
					const int pending = __syncthreads_count(need ? 1 : 0);
					front = S.front[it & 1];
					nlive = S.nlive[it & 1];
#ifdef B200Z_DEBUG_PASSES
					if (tid == 0) printf("  pass %d: pending %d live %u front %d lastlane %d\n", it, pending, nlive, front, lastlane);
#endif
					if (!pending) break;
				}
				if (tid == 0) {
					atomicAdd(&ctr->n_rounds, 1u);
					atomicAdd(&ctr->n_passes, passes);
				}
				// lanes up to and including the first one that stopped the block are exact; the rest are dead
				if (tid > lastlane) {
					obytes = 0;
					nmatch = 0;
				}
				// exclusive prefix sums over the 128 lanes
				uint32_t io = obytes, im = nmatch;
				for (int o = 1; o < 32; o <<= 1) {
					const uint32_t t1 = __shfl_up_sync(0xffffffffu, io, o);
					const uint32_t t2 = __shfl_up_sync(0xffffffffu, im, o);
					if (lane >= o) {
						io += t1;
						im += t2;
					}
				}
				if (lane == 31) {
					S.wsum_o[warp] = io;
					S.wsum_m[warp] = im;
				}
				__syncthreads();
				uint32_t bo = 0, bm = 0, tot = 0, totm = 0;
				for (int w = 0; w < kP1Threads / 32; w++) {
					if (w < warp) {
						bo += S.wsum_o[w];
						bm += S.wsum_m[w];
					}
					tot += S.wsum_o[w];
					totm += S.wsum_m[w];
				}
				const uint32_t lflags = S.flags[lastlane], ldet = S.dets[lastlane], lexit = S.exitp[lastlane];
				if (batch_used == kRoundBatch) {
					if (tid == 0) S.a_base = atomicAdd(&ctr->round_top, (uint32_t)kRoundBatch);
					__syncthreads();
					batch_base = S.a_base;
					batch_used = 0;
					if (batch_base + kRoundBatch > round_cap) {
						end_kind = SEG_POOL;
						break;
					}
					if (tid < kRoundBatch) rounds[batch_base + tid].kind = RND_NONE;
					__syncthreads();
				}
				{
					PRound &r = rounds[batch_base + batch_used];
					r.entry[tid] = entry;
					r.opre[tid] = bo + io - obytes;
					r.mpre[tid] = bm + im - nmatch;
					if (tid == 0) {
						r.seg = slot;
						r.hdr = hdr_idx;
						r.w0 = w0;
						r.r0 = r0;
						r.end_rel = end_rel;
						r.lastlane = (uint32_t)lastlane;
						r.nbytes = tot;
						r.out_rel = opos;
						r.match_rel = nm_total;
						r.kind = RND_HUFF;
					}
					++batch_used;
				}
				opos += tot;
				nm_total += totm;
				bitpos = ((uint64_t)w0 << 5) + lexit;
				if (lflags & F_EOB) in_block = false;
				else if (lflags & F_OVERRUN) { st = B200Z_E_NEED_INPUT; in_block = false; }
				else if (lflags & F_ERR) { st = B200Z_E_DATA; detail = (int)ldet; in_block = false; }
				else if (tot == 0 && lexit == r0) { st = B200Z_E_INTERNAL; in_block = false; } // cannot happen: a symbol always fits
			}
			if (st != B200Z_OK || end_kind == SEG_POOL) break;
			++blocks_done;
		}
		if (tid == 0) {
			seg.end_bit = bitpos;
			seg.rs_bit = rs_bit;
			seg.body_bit = S.h_body;
			seg.rs_out = rs_out;
			seg.out_bytes = opos;
			seg.n_match = nm_total;
			seg.end_kind = end_kind;
			seg.status = st | (detail << 8);
		}
	}
}

// ---------------------------------------------------------------------------------------------------------
// k_chain: one thread per stream
// ---------------------------------------------------------------------------------------------------------
__global__ void k_chain(int n, PSeg *__restrict__ segs, const uint32_t *__restrict__ win_base, const int64_t *__restrict__ in_len,
                        const int64_t *__restrict__ out_cap, const uint32_t *__restrict__ match_cap, const int32_t *__restrict__ pre,
                        int64_t *__restrict__ out_len, int64_t *__restrict__ in_used, int32_t *__restrict__ status,
                        int64_t *__restrict__ restart, uint32_t *__restrict__ str_nm, int32_t *__restrict__ fallback) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	fallback[i] = 0;
	str_nm[i] = 0;
	if (pre && pre[i] != B200Z_OK) { // the framing header was rejected (k_wrap_head): nothing to decode
		status[i] = pre[i];
		out_len[i] = 0;
		if (in_used) in_used[i] = 0;
		put_restart(restart, i, 0, 0, 0, 0, 0);
		return;
	}
	const uint32_t wb = win_base[i];
	uint64_t out = 0, nm = 0;
	uint32_t cur = (uint32_t)i;
	int st = B200Z_OK;
	uint64_t end_bit = 0, rs_bit = 0, rs_out = 0, body_bit = 0;
	bool pool = false;
	// pass 1: totals
	for (;;) {
		const PSeg &s = segs[cur];
		rs_bit = s.rs_bit;
		rs_out = out + s.rs_out;
		body_bit = s.body_bit;
		out += s.out_bytes;
		nm += s.n_match;
		end_bit = s.end_bit;
		if (s.end_kind == SEG_JOIN) {
			cur = (uint32_t)n + wb + (uint32_t)(s.end_bit >> kFWShift);
			continue;
		}
		if (s.end_kind == SEG_POOL) pool = true;
		else if (s.end_kind == SEG_FINAL) st = B200Z_OK;
		else st = s.status;
		break;
	}
	if (pool || out > 0xFFFF0000ull || nm > (uint64_t)match_cap[i]) {
		fallback[i] = 1; // the serial kernel decodes this stream
		return;
	}
	if (out > (uint64_t)out_cap[i]) {
		status[i] = B200Z_E_NOMEM;
		out_len[i] = 0;
		if (in_used) in_used[i] = 0;
		const uint64_t sb = segs[i].start_bit;
		put_restart(restart, i, sb, 0, sb, sb, 0);
		return;
	}
	// pass 2: positions
	cur = (uint32_t)i;
	uint64_t o = 0;
	uint32_t m = 0;
	for (;;) {
		PSeg &s = segs[cur];
		s.out_base = o;
		s.match_base = m;
		s.valid = 1;
		o += s.out_bytes;
		m += s.n_match;
		if (s.end_kind != SEG_JOIN) break;
		cur = (uint32_t)n + wb + (uint32_t)(s.end_bit >> kFWShift);
	}
	status[i] = st;
	out_len[i] = (int64_t)out;
	str_nm[i] = (uint32_t)nm;
	if (in_used) {
		uint64_t used = (end_bit + 7) >> 3; // n - RemainingInput (trap T14)
		if (used > (uint64_t)in_len[i]) used = (uint64_t)in_len[i];
		in_used[i] = (int64_t)used;
	}
	const bool mid = (st & 0xFF) == B200Z_E_NEED_INPUT && body_bit != rs_bit; // the input ended inside a Huffman block
	put_restart(restart, i, rs_bit, rs_out, mid ? body_bit : rs_bit, mid ? end_bit : rs_bit, mid ? out : rs_out);
}

// ---------------------------------------------------------------------------------------------------------
// k_dec2: the final decode pass, one CTA per batch of rounds
// ---------------------------------------------------------------------------------------------------------
struct __align__(16) Dec2Shared {
	InfShared sh;
	uint32_t in[2][kP1InSlots]; // the round being decoded and the next one, staged with asynchronous copies meanwhile
};

// a round's words into shared memory, 4 bytes per asynchronous copy (LDGSTS): nobody waits for them here
__device__ __forceinline__ void stage_round_async(uint32_t *words, const uint32_t *gwords, uint32_t w0, uint32_t nwords) {
	for (int i = threadIdx.x; i < kP1InWords; i += blockDim.x) {
		const uint32_t wi = w0 + (uint32_t)i;
		// (bytes behind the stream's end inside its last word are never looked at: every symbol is checked against end_rel)
		if (wi < nwords) __pipeline_memcpy_async(&words[in_slot((uint32_t)i)], gwords + wi, 4);
		else words[in_slot((uint32_t)i)] = 0;
	}
	__pipeline_commit();
}

__global__ void __launch_bounds__(kP1Threads)
    k_dec2(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
           const int64_t *__restrict__ out_off, const PSeg *__restrict__ segs, const PCounters *__restrict__ ctr,
           const PRound *__restrict__ rounds, uint32_t round_cap, const PBlockHdr *__restrict__ hdrs, MatchTok *__restrict__ mlist,
           const int64_t *__restrict__ mt_off) {
	extern __shared__ __align__(16) uint8_t smem_raw[];
	Dec2Shared &S = *reinterpret_cast<Dec2Shared *>(smem_raw);
	const int tid = threadIdx.x;
	uint32_t top = ctr->round_top;
	if (top > round_cap) top = round_cap;
	for (uint32_t b0 = blockIdx.x * kRoundBatch; b0 < top; b0 += gridDim.x * kRoundBatch) {
		// a batch holds the rounds of ONE block of one segment (or one stored block in its first slot)
		const PRound &r0 = rounds[b0];
		if (r0.kind == RND_NONE) continue;
		const PSeg &seg = segs[r0.seg];
		if (!seg.valid) continue;
		const uint32_t stream = seg.stream;
		uint8_t *dst = out + out_off[stream];
		if (r0.kind == RND_STORED) {
			const uint8_t *src = in + in_off[stream] + r0.w0;
			const uint64_t obase = seg.out_base + r0.out_rel;
			const uint32_t len = r0.nbytes;
			for (uint32_t i = tid; i < len; i += kP1Threads) dst[obase + i] = src[i];
			continue;
		}
		const uint32_t nbytes = (uint32_t)in_len[stream], nwords = (nbytes + 3) >> 2;
		const uint32_t *gwords = reinterpret_cast<const uint32_t *>(in + in_off[stream]);
		int nr = 1;
		while (nr < kRoundBatch && rounds[b0 + nr].kind == RND_HUFF) ++nr;
		__syncthreads(); // the previous batch's lanes are done with the tables and the staged words
		stage_round_async(S.in[0], gwords, r0.w0, nwords);
		{
			const uint4 *src = reinterpret_cast<const uint4 *>(&hdrs[r0.hdr].tab);
			uint4 *dstv = reinterpret_cast<uint4 *>(&S.sh);
			for (int i = tid; i < (int)(sizeof(InfShared) / 16); i += kP1Threads) dstv[i] = src[i];
		}
		for (int k = 0; k < nr; k++) {
			const PRound &r = rounds[b0 + k];
			const uint32_t *words = S.in[k & 1];
			if (k + 1 < nr) {
				stage_round_async(S.in[(k + 1) & 1], gwords, rounds[b0 + k + 1].w0, nwords); // (its last readers left at the barrier below)
				__pipeline_wait_prior(1);
			} else {
				__pipeline_wait_prior(0);
			}
			__syncthreads(); // round k's words (and, for k = 0, the tables) are in place
			{
				const bool mine = (uint32_t)tid <= r.lastlane;
				SpanB sp;
				span_begin(sp, words, mine ? r.entry[tid] : 0u);
				const uint32_t lim = r.r0 + (uint32_t)(tid + 1) * kSubBits;
				const uint64_t o0 = seg.out_base + r.out_rel + (mine ? r.opre[tid] : 0u);
				MatchTok *ml = mlist + mt_off[stream] + seg.match_base + r.match_rel + (mine ? r.mpre[tid] : 0u);
				const uint32_t end_rel = r.end_rel;
				// warp-synchronous: the lanes step together and re-converge every symbol
				bool act = mine;
				while (__any_sync(0xffffffffu, act)) {
					if (act) act = span_step2<1>(S.sh, words, sp, lim, end_rel, dst, o0, ml);
					__syncwarp();
				}
			}
			__syncthreads(); // everybody is done with round k's words: the round after next may overwrite them
		}
	}
}

// ---------------------------------------------------------------------------------------------------------
// k_resolve: back-references, one CTA per stream, 16 KiB tiles in stream order.  The last 64 KiB of the stream's output
// live in a shared-memory ring (ring[a & 65535] = output byte a; bytes in front of the stream: the preset dictionary's
// tail, else zeros -- a fresh reference window holds zeros, trap T13), so every source byte of a back-reference is a
// shared-memory read: sources in front of the tile are final, sources inside the tile are resolved by pointer jumping.
// ---------------------------------------------------------------------------------------------------------
constexpr int kResRing = 65536;
constexpr int kResChunk = 2048; // back-references a tile may hold: a tile ends early where the 2048th would start
struct __align__(16) ResShared {
	uint8_t ring[kResRing];
	// per byte of the tile: first a mark (index + 1 of the back-reference that STARTS here, 0 = none), then the ring index of
	// the byte it is a copy of (its own: a literal), after jumps of a byte further back
	uint16_t ptr[kResTile];
	MatchTok mch[kResChunk];
	uint32_t wmax[kResThreads / 32];
	int cnt_in, cnt_done;
};

__global__ void __launch_bounds__(kResThreads, 2) // two CTAs per SM: 32 registers per thread
    k_resolve(const uint8_t *__restrict__ in, uint8_t *out, const int64_t *__restrict__ in_off, const int64_t *__restrict__ out_off,
              const uint32_t *__restrict__ dict_len, const int64_t *__restrict__ out_len, const uint32_t *__restrict__ str_nm,
              const int32_t *__restrict__ fallback, const MatchTok *__restrict__ mlist, const int64_t *__restrict__ mt_off, int n) {
	extern __shared__ __align__(16) uint8_t smem_raw[];
	ResShared &S = *reinterpret_cast<ResShared *>(smem_raw);
	const int stream = blockIdx.x;
	if (stream >= n || fallback[stream]) return;
	const uint32_t nm = str_nm[stream];
	if (nm == 0) return; // no back-reference: the literals are in place
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	uint8_t *dst = out + out_off[stream];
	const int64_t total = out_len[stream];
	const MatchTok *ml = mlist + mt_off[stream];
	{
		// what lies in front of the stream: ring[65536 - k] = byte -k
		const uint32_t D = dict_len[stream];
		const uint8_t *dict = in + in_off[stream] - D; // the preset dictionary's tail lies in front of the compressed bytes
		for (int i = tid; i < kResRing / 2; i += kResThreads) {
			const int k = kResRing / 2 - i; // 32768 .. 1 bytes in front of position 0
			S.ring[kResRing - k] = (uint32_t)k <= D ? dict[D - (uint32_t)k] : (uint8_t)0;
		}
	}
	uint32_t cur_m = 0;
	const uint4 zero4 = make_uint4(0, 0, 0, 0);
	MatchTok none;
	none.out_pos = 0xFFFFFFFFu;
	none.len = 0;
	none.dist = 0;
	// software pipeline: the next tile's bytes (as k_dec2 left them: literals in place) and the next tile's
	// back-references are loaded while the current tile is resolved
	const int a0 = tid * 16; // the 16 consecutive bytes this thread loads, sets up and stores (jumps: bytes tid + 1024 k)
	uint4 nxt_tile = zero4;
	if ((int64_t)a0 + 16 <= total) nxt_tile = *reinterpret_cast<const uint4 *>(dst + a0);
	int64_t nxt_at = 0; // the position nxt_tile was loaded for
	MatchTok nxt_m0 = (uint32_t)tid < nm ? ml[tid] : none, nxt_m1 = (uint32_t)(kResThreads + tid) < nm ? ml[kResThreads + tid] : none;
	for (int64_t T0 = 0; T0 < total;) { // T0 stays a multiple of 16
		int tl = (int)(total - T0 < (int64_t)kResTile ? total - T0 : (int64_t)kResTile);
		const uint32_t rbase = (uint32_t)T0 & (uint32_t)(kResRing - 1);
		__syncthreads(); // the previous tile is resolved and written back
		if (nxt_at != T0) nxt_tile = (int64_t)T0 + a0 + 16 <= total ? *reinterpret_cast<const uint4 *>(dst + T0 + a0) : zero4; // (behind a short tile)
		if (a0 + 16 <= tl) {
			*reinterpret_cast<uint4 *>(S.ring + ((rbase + (uint32_t)a0) & (uint32_t)(kResRing - 1))) = nxt_tile;
		} else {
			for (int i = a0; i < tl && i < a0 + 16; i++) S.ring[(rbase + (uint32_t)i) & (uint32_t)(kResRing - 1)] = dst[T0 + i];
		}
		{
			nxt_at = T0 + kResTile;
			const int64_t a = nxt_at + (int64_t)a0;
			nxt_tile = a + 16 <= total ? *reinterpret_cast<const uint4 *>(dst + a) : zero4;
		}
		if (cur_m >= nm) break; // nothing left to resolve (the remaining tiles are literals only)
		// ---- the back-references that reach into the tile ----
		if (tid == 0) {
			S.cnt_in = 0;
			S.cnt_done = 0;
		}
		for (int i = tid; i < kResTile / 2; i += kResThreads) reinterpret_cast<uint32_t *>(S.ptr)[i] = 0; // no marks
		S.mch[tid] = nxt_m0;
		S.mch[kResThreads + tid] = nxt_m1;
		__syncthreads();
		int64_t T1 = T0 + tl;
		{
			// a full chunk whose last reference still starts inside the tile: the tile ends (16-byte aligned) in front of it
			const MatchTok lastm = S.mch[kResChunk - 1];
			if (cur_m + (uint32_t)kResChunk <= nm && (int64_t)lastm.out_pos < T1) {
				T1 = (int64_t)lastm.out_pos & ~15ll; // > T0: 2047 references in front of it cover more than 6 KiB
				tl = (int)(T1 - T0);
			}
		}
		{
			const uint32_t mi0 = cur_m + (uint32_t)tid, mi1 = cur_m + (uint32_t)(kResThreads + tid);
			int ci = 0, cd = 0;
			// a back-reference marks its first byte in the tile with its index in the chunk + 1
			if (mi0 < nm && (int64_t)nxt_m0.out_pos < T1) {
				ci++;
				cd += (int64_t)nxt_m0.out_pos + nxt_m0.len <= T1;
				const int64_t dl = (int64_t)nxt_m0.out_pos - T0;
				S.ptr[dl > 0 ? dl : 0] = (uint16_t)(tid + 1);
			}
			if (mi1 < nm && (int64_t)nxt_m1.out_pos < T1) {
				ci++;
				cd += (int64_t)nxt_m1.out_pos + nxt_m1.len <= T1;
				const int64_t dl = (int64_t)nxt_m1.out_pos - T0;
				S.ptr[dl > 0 ? dl : 0] = (uint16_t)(kResThreads + tid + 1);
			}
			for (int o = 16; o > 0; o >>= 1) {
				ci += __shfl_xor_sync(0xffffffffu, ci, o);
				cd += __shfl_xor_sync(0xffffffffu, cd, o);
			}
			if (lane == 0 && ci) {
				atomicAdd(&S.cnt_in, ci);
				atomicAdd(&S.cnt_done, cd);
			}
		}
		__syncthreads();
		const int n_in = S.cnt_in;
		cur_m += (uint32_t)S.cnt_done;
		{
			const uint32_t ni0 = cur_m + (uint32_t)tid, ni1 = cur_m + (uint32_t)(kResThreads + tid);
			nxt_m0 = ni0 < nm ? ml[ni0] : none;
			nxt_m1 = ni1 < nm ? ml[ni1] : none;
		}
		if (n_in == 0) { // no back-reference touches this tile
			T0 = T1;
			continue;
		}
		// Which back-reference covers a byte: the last one that starts at or in front of it -- a running maximum over the
		// marks (they grow with the position).  Every thread scans its 16 consecutive bytes, the threads' totals are scanned
		// over the warp and the CTA, then every byte turns its owner into the ring index of its source (OutputWindow.Repeat:
		// byte k of a copy comes from source byte k mod distance) -- a literal into its own.
		const uint4 mlo = *reinterpret_cast<const uint4 *>(S.ptr + a0), mhi = *reinterpret_cast<const uint4 *>(S.ptr + a0 + 8);
		uint32_t before;
		{
			const uint32_t w[8] = {mlo.x, mlo.y, mlo.z, mlo.w, mhi.x, mhi.y, mhi.z, mhi.w};
			uint32_t run = 0;
#pragma unroll
			for (int k = 0; k < 8; k++) {
				const uint32_t lo16 = w[k] & 0xFFFFu, hi16 = w[k] >> 16;
				run = lo16 > run ? lo16 : run;
				run = hi16 > run ? hi16 : run;
			}
			uint32_t incl = run;
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
				if (lane >= o && t > incl) incl = t;
			}
			if (lane == 31) S.wmax[warp] = incl;
			before = __shfl_up_sync(0xffffffffu, incl, 1);
			if (lane == 0) before = 0;
		}
		__syncthreads();
		for (int w = 0; w < warp; w++) {
			const uint32_t t = S.wmax[w];
			before = t > before ? t : before;
		}
		{
			const uint32_t w[8] = {mlo.x, mlo.y, mlo.z, mlo.w, mhi.x, mhi.y, mhi.z, mhi.w};
			uint32_t res[8];
			uint32_t run = before;
#pragma unroll
			for (int k = 0; k < 16; k++) {
				const uint32_t mark = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
				run = mark > run ? mark : run;
				const int p = a0 + k;
				uint32_t val = (rbase + (uint32_t)p) & 0xFFFFu; // a literal: its own source
				if (run) {
					const MatchTok g = S.mch[run - 1];
					const int dl = (int)((int64_t)g.out_pos - T0); // may be negative: the reference started in the previous tile
					const int kk = p - dl;
					if (kk < (int)g.len) {
						const int dist = g.dist ? (int)g.dist : 65536; // (never 0 for a decoded back-reference)
						const int so = dist >= (int)g.len ? kk : kk % dist;
						val = (rbase + (uint32_t)(dl - dist + so)) & 0xFFFFu;
					}
				}
				if (k & 1) res[k >> 1] |= val << 16;
				else res[k >> 1] = val;
			}
			*reinterpret_cast<uint4 *>(S.ptr + a0) = make_uint4(res[0], res[1], res[2], res[3]);
			*reinterpret_cast<uint4 *>(S.ptr + a0 + 8) = make_uint4(res[4], res[5], res[6], res[7]);
		}
		__syncthreads();
		// pointer jumping: a byte takes over its source's source until that is a final byte (one in front of the tile, or a
		// literal of the tile, which is its own source).  Bytes tid + 1024 k: the warp's accesses are consecutive.
		uint32_t live = 0xFFFFu;
		for (;;) {
			int changed = 0;
#pragma unroll
			for (int k = 0; k < 16; k++) {
				if (!((live >> k) & 1u)) continue;
				const int i = tid + k * kResThreads;
				bool keep = false;
				if (i < tl) {
					const uint32_t q = S.ptr[i];
					const uint32_t ql = (q - rbase) & (uint32_t)(kResRing - 1);
					if (ql < (uint32_t)tl && ql != (uint32_t)i) {
						const uint32_t r = S.ptr[ql];
						if (r != q) {
							S.ptr[i] = (uint16_t)r;
							changed = 1;
							keep = true;
						}
					}
				}
				if (!keep) live &= ~(1u << k);
			}
			if (!__syncthreads_or(changed)) break;
		}
		// the tile's bytes: copies fetch their final source; into the ring and out (nobody's pointer ends on a copy)
		if (a0 + 16 <= tl) {
			const uint4 lo = *reinterpret_cast<const uint4 *>(S.ptr + a0), hi = *reinterpret_cast<const uint4 *>(S.ptr + a0 + 8);
			const uint32_t pw[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
			uint32_t w[4];
#pragma unroll
			for (int q = 0; q < 4; q++) {
				uint32_t x = 0;
#pragma unroll
				for (int b2 = 0; b2 < 4; b2++) {
					const int k = q * 4 + b2;
					x |= (uint32_t)S.ring[(pw[k >> 1] >> (16 * (k & 1))) & 0xFFFFu] << (8 * b2);
				}
				w[q] = x;
			}
			const uint4 v = make_uint4(w[0], w[1], w[2], w[3]);
			*reinterpret_cast<uint4 *>(S.ring + ((rbase + (uint32_t)a0) & (uint32_t)(kResRing - 1))) = v;
			*reinterpret_cast<uint4 *>(dst + T0 + a0) = v;
		} else {
			for (int i = a0; i < tl && i < a0 + 16; i++) {
				const uint8_t x = S.ring[S.ptr[i]];
				S.ring[(rbase + (uint32_t)i) & (uint32_t)(kResRing - 1)] = x;
				dst[T0 + i] = x;
			}
		}
		T0 = T1;
	}
}

} // namespace b200z
