// b200z_deflate.cu -- the sm_90a DEFLATE compressor for the reference's lazy levels (5-9).
// Kernel decomposition and the reference lines each kernel replaces: see b200z_core.cuh and DESIGN.md.
//
//   k_links   (K1)  DeflaterEngine.InsertString / head[] / prev[]         DeflaterEngine.cs:417-439
//   k_match   (K2)  DeflaterEngine.FindLongestMatch, for every position   DeflaterEngine.cs:474-612
//   k_parse   (K3)  DeflaterEngine.DeflateSlow state machine              DeflaterEngine.cs:741-855
//   k_plan    (K4)  DeflaterHuffman.FlushBlock up to the type decision    DeflaterHuffman.cs:788-857
//   k_scan    (K5)  bit position of every block; Deflater flush padding   Deflater.cs:486-517
//   k_emit    (K6)  SendAllTrees / CompressBlock / FlushStoredBlock       DeflaterHuffman.cs:676-779
#include <cuda_pipeline.h>

#include <memory>

#include "b200z_internal.cuh"
#include "b200z_tma.cuh"

namespace b200z {

constexpr int kRun = 65536;    // positions per k_links warp
constexpr int kTile = 32768;   // positions per k_match CTA
constexpr int kTileData = 2 * kTile + 320; // bytes of window staged per tile (history + tile + max match + pad)
constexpr int kMatchThreads = 1024;
constexpr int kMatchClasses = 16; // expected-walk-length classes of k_match (0 = nothing to search)

// ------------------------------------------------------------------------------------------------
// K1: link[p] = distance from p to the previous inserted position with the same hash (0 = none / too far).
// One warp per run of kRun positions, 32 positions per step; a 16-bit head table in shared memory, re-based
// every 32768 positions exactly like SlideWindow (DeflaterEngine.cs:441-462) so that entries stay unambiguous.
// ------------------------------------------------------------------------------------------------
// lanes holding the same 15-bit hash, from 16 ballots (MATCH.ANY showed ~360 cycles of latency per step in ncu)
__device__ __forceinline__ uint32_t same_hash_mask(uint32_t h, bool valid, int lane) {
	uint32_t eq = __ballot_sync(0xffffffffu, valid);
#pragma unroll
	for (int b = 0; b < 15; b++) {
		const bool bit = (h >> b) & 1u;
		const uint32_t bal = __ballot_sync(0xffffffffu, bit);
		eq &= bit ? bal : ~bal;
	}
	return valid ? eq : (1u << lane);
}

// The head table is a serial dependency chain (every step reads what the previous step wrote), so the CTA splits the work:
// four PRODUCER warps compute, for groups of 32 positions, everything that does not depend on the table -- hash, validity,
// the nearest lower lane with the same hash, whether the lane is the last of its hash in the group -- and leave one word
// per position in shared memory; the CONSUMER warp then only does  read word -> read head -> write head -> store link.
// ncu before the split: one warp did both, ~570 cycles per step, 4 % of the SM's warp slots occupied.
constexpr int kLinkChunk = 512;                   // positions per hand-over between producers and consumer
constexpr int kLinkProducers = 8;
constexpr int kLinkThreads = 32 * (1 + kLinkProducers); // warp 0 consumes, the others produce
constexpr int kLinkRebase = 16384;                // head entries are re-based this often (see below)
constexpr int kLinksSmem = 65536 + 2 * kLinkChunk * 4;

__global__ void __launch_bounds__(kLinkThreads) k_links(const uint8_t *__restrict__ in, uint16_t *__restrict__ link,
                                                        const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                                                        const int2 *__restrict__ run_desc, const uint32_t *__restrict__ hist,
                                                        const uint8_t *__restrict__ hmask, const int64_t *__restrict__ hm_off,
                                                        uint32_t run_len) {
	extern __shared__ __align__(16) uint8_t lsm[];
	uint16_t *head = reinterpret_cast<uint16_t *>(lsm);             // 32768 entries: position - winbase + 1, 0 = empty
	uint32_t *info = reinterpret_cast<uint32_t *>(lsm + 65536);     // two buffers of kLinkChunk words
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int2 rd = run_desc[blockIdx.x];
	const uint32_t n = (uint32_t)in_len[rd.x];
	const uint8_t *data = in + in_off[rd.x];
	uint16_t *lnk = link + in_off[rd.x];
	const uint32_t start = (uint32_t)rd.y;
	const uint32_t run_end = (n - start > run_len) ? start + run_len : n; // run_len: kRun, or what B200Z_LINK_RUN asked for
	const uint32_t warm = start >= 32768u ? start - 32768u : 0u;
	// history (preset dictionary / earlier segments of the same stream): positions the reference never inserted
	// (the last two of a dictionary, DeflaterEngine.cs:217-226, or of a flushed segment, trap T9) are masked
	const uint32_t H = hist[rd.x];
	const uint8_t *hm = hmask + hm_off[rd.x];
	for (int i = threadIdx.x; i < 16384; i += kLinkThreads) reinterpret_cast<uint32_t *>(head)[i] = 0;
	uint32_t winbase = warm;
	auto produce = [&](uint32_t cb, int which) {
		// all of the warp's loads first (they are independent), then the ballots
		constexpr int G = kLinkChunk / 32 / kLinkProducers; // groups per producer warp and chunk
		uint32_t hh[G];
		bool vv[G];
#pragma unroll
		for (int j = 0; j < G; j++) {
			const uint32_t p = cb + 32u * (uint32_t)(warp - 1 + kLinkProducers * j) + lane;
			bool valid = p + 2 < n; // InsertString only while lookahead >= MIN_MATCH (DeflaterEngine.cs:782, :819)
			uint32_t h = 0;
			if (p + 2 < n) h = hash3(__ldg(data + p), __ldg(data + p + 1), __ldg(data + p + 2));
			if (p < H && valid) valid = __ldg(hm + p) == 0;
			hh[j] = h;
			vv[j] = valid;
		}
#pragma unroll
		for (int j = 0; j < G; j++) {
			const uint32_t g = (uint32_t)(warp - 1 + kLinkProducers * j);
			if (cb + 32u * g >= run_end) break;
			const uint32_t h = hh[j];
			const bool valid = vv[j];
			const uint32_t mask = same_hash_mask(h, valid, lane);
			const uint32_t lower = mask & ((1u << lane) - 1u);
			uint32_t w = h;
			if (valid) {
				w |= 1u << 15;
				if (lower) w |= (1u << 16) | ((uint32_t)(31 - __clz(lower)) << 17);
				if ((mask >> lane) == 1u) w |= 1u << 22;
			}
			info[which * kLinkChunk + 32u * g + lane] = w;
		}
	};
	if (warp > 0) produce(warm, 0);
	__syncthreads();
	int which = 0;
	for (uint32_t cb = warm; cb < run_end; cb += kLinkChunk, which ^= 1) {
		// The 16-bit entries are kept unambiguous like SlideWindow does (DeflaterEngine.cs:441-462), but in steps of 16384:
		// before a chunk starting 49152 or more past winbase, every entry drops by 16384 and entries that cannot be
		// within MAX_DIST of any position still to come (older than cb - 32768) vanish.  Which entries survive beyond
		// MAX_DIST is irrelevant: link[] only keeps distances <= MAX_DIST.
		if (cb - winbase >= 49152u) {
			for (int i = threadIdx.x; i < 16384; i += kLinkThreads) {
				uint32_t v = reinterpret_cast<uint32_t *>(head)[i];
				uint32_t lo = v & 0xFFFFu, hi = v >> 16;
				lo = lo > (uint32_t)kLinkRebase ? lo - kLinkRebase : 0u;
				hi = hi > (uint32_t)kLinkRebase ? hi - kLinkRebase : 0u;
				reinterpret_cast<uint32_t *>(head)[i] = lo | (hi << 16);
			}
			winbase += kLinkRebase;
			__syncthreads();
		}
		if (warp == 0) {
			const uint32_t cend = (run_end - cb > (uint32_t)kLinkChunk) ? cb + kLinkChunk : run_end;
			const uint32_t *ib = info + which * kLinkChunk;
			uint32_t w = ib[lane];
			for (uint32_t base = cb; base < cend; base += 32) {
				const uint32_t p = base + lane;
				const uint32_t wn = ib[(base + 32 - cb + lane) & (kLinkChunk - 1)]; // next group's word (unused after the last)
				// branch-free: every lane reads head[h] (h = 0 for lanes without a hash), the selects sort it out
				const uint32_t h = w & 0x7FFFu;
				const uint32_t v = head[h];
				const bool valid = (w >> 15) & 1u;
				uint32_t q = v ? winbase + v - 1 : 0xFFFFFFFFu;
				if ((w >> 16) & 1u) q = base + ((w >> 17) & 31u);
				__syncwarp();
				if (valid && ((w >> 22) & 1u)) head[h] = (uint16_t)(p - winbase + 1);
				__syncwarp();
				const uint32_t d = (valid && q != 0xFFFFFFFFu) ? p - q : 0u;
				if (p >= start && p < run_end) lnk[p] = (d <= (uint32_t)kMaxDist) ? (uint16_t)d : (uint16_t)0;
				w = wn;
			}
		} else if (cb + kLinkChunk < run_end) {
			produce(cb + kLinkChunk, which ^ 1);
		}
		__syncthreads();
	}
}

// ------------------------------------------------------------------------------------------------
// K2: per-position match table.  One CTA per 32 KiB tile; the tile's 64 KiB data window and the window's link
// entries are staged in shared memory (192 KiB), then each thread walks the chains of 32 positions.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kMatchThreads, 1)
    k_match(const uint8_t *__restrict__ in, const uint16_t *__restrict__ link, uint2 *__restrict__ mt,
            const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len, const int2 *__restrict__ tile_desc,
            const uint32_t *__restrict__ hist, const int64_t *__restrict__ bias, uint32_t *__restrict__ scratch, LevelParams lp) {
	extern __shared__ __align__(16) uint8_t smem[];
	uint8_t *s_data = smem;
	uint16_t *s_link = reinterpret_cast<uint16_t *>(smem + kTileData);
	const int2 td = tile_desc[blockIdx.x];
	const uint32_t n = (uint32_t)in_len[td.x];
	const int64_t off = in_off[td.x];
	const uint8_t *data = in + off;
	const uint16_t *lnk = link + off;
	const uint32_t t0 = (uint32_t)td.y;
	const uint32_t t1 = (n - t0 > (uint32_t)kTile) ? t0 + kTile : n;
	const uint32_t w0 = t0 >= (uint32_t)kTile ? t0 - kTile : 0u;
	uint32_t dend = t1 + 272;
	if (dend > n) dend = n;
	// Stage the tile's 64 KiB data window and its link entries (w0 and the slot base are 16-byte aligned).  The bulk of both
	// goes through the TMA engine: one thread arms an mbarrier with the byte count and issues cp.async.bulk copies, the
	// CTA waits on the barrier; the tails that are not multiples of 16 bytes are covered by scalar loops meanwhile.
	__shared__ BulkBarrier s_bar;
	if (threadIdx.x == 0) bulk_barrier_init(&s_bar);
	__syncthreads();
	{
		const uint32_t nbytes = dend - w0;
		const uint32_t nvec = nbytes >> 4;
		const uint32_t nl = t1 - w0;
		const uint32_t nlv = nl >> 3;
		if (threadIdx.x == 0) {
			bulk_expect(&s_bar, 16u * (nvec + nlv));
			bulk_copy_start(&s_bar, s_data, data + w0, 16u * nvec);
			bulk_copy_start(&s_bar, s_link, lnk + w0, 16u * nlv);
		}
		for (uint32_t i = (nvec << 4) + threadIdx.x; i < nbytes; i += kMatchThreads) s_data[i] = data[w0 + i];
		for (uint32_t i = (nlv << 3) + threadIdx.x; i < nl; i += kMatchThreads) s_link[i] = lnk[w0 + i];
	}
	bulk_wait(&s_bar, 0);
	__syncthreads();
	// "No predecessor" (0) becomes a jump of 0xFFFF window positions: it lands below any position's lowest chain index
	// (more than kMaxDist back), so one compare ends a walk at the chain's end and at the distance limit alike.
	{
		uint32_t *s_lw = reinterpret_cast<uint32_t *>(s_link);
		const uint32_t nw = (t1 - w0 + 1) >> 1; // an odd count also rewrites the slot behind the last one: never staged, never read
		for (uint32_t i = threadIdx.x; i < nw; i += kMatchThreads) {
			uint32_t w = s_lw[i];
			if ((w & 0xFFFFu) == 0) w |= 0xFFFFu;
			if ((w >> 16) == 0) w |= 0xFFFF0000u;
			s_lw[i] = w;
		}
	}
	__syncthreads();
	uint2 *out = mt + off;
	// match_search() of b200z_core.cuh with the byte-wise extension loop replaced by 4-byte compares on aligned
	// shared-memory words (ncu: the byte loop ran with ~2 of 32 lanes active and took ~30 % of the kernel).
	const uint32_t chain = (uint32_t)lp.chain, budgetB = chain >> 2;
	const uint32_t H = hist[td.x];            // positions below H are history: candidates only
	const uint32_t ab = (uint32_t)bias[td.x]; // absolute stream offset of buffer position 0 (window-slide phase, trap T8)
	// ---- order the tile's positions by expected chain length ----
	// A warp runs as long as its longest chain walk (ncu: 13 of 32 lanes active in the candidate loop).  So the positions
	// are bucketed by an estimate of their walk length (the first eight hops are exact, beyond that their hop density
	// extrapolated over the window) and handed to the threads longest first: warps then hold walks of similar length.
	// The order only decides who computes what; every position's result is unchanged.
	// (Tried and dropped: the walks as a flat state machine -- one candidate test or four bytes of extension per lane and
	// iteration, free lanes refilled from the ordered list eight at a time.  Bit-exact but slower on the bench workload:
	// every iteration pays for every state's code.)
	__shared__ uint32_t s_cls[2][kMatchClasses];
	if (threadIdx.x < 2 * kMatchClasses) (&s_cls[0][0])[threadIdx.x] = 0;
	__syncthreads();
	uint16_t *order = reinterpret_cast<uint16_t *>(scratch + off + t0); // 4 bytes per position are free here until k_parse_gather
	uint32_t cw[4] = {0u, 0u, 0u, 0u};                                   // 32 x 4 bits: this thread's classes
	const int lane = threadIdx.x & 31;
#pragma unroll
	for (int k = 0; k < kTile / kMatchThreads; k++) {
		const uint32_t p = t0 + threadIdx.x + (uint32_t)k * kMatchThreads;
		uint32_t cls = 0;
		if (p < t1 && p >= H) {
			const uint32_t la = n - p;
			uint32_t d = la >= (uint32_t)kMinMatch ? (uint32_t)s_link[p - w0] : 0u;
			if (d > (uint32_t)kMaxDist - (is_slide_pos(p + ab) ? 1u : 0u)) d = 0; // DeflaterEngine.cs:788 + trap T8
			if (d == 0) out[p] = make_uint2(0u, 0u);
			else {
				const uint32_t is = p - w0;
				uint32_t dist = d, hops = 1;
				while (hops < 8) {
					const uint32_t l2 = s_link[is - dist];
					if (dist + l2 >= (uint32_t)kMaxDist) break; // also the chain's end (0xFFFF)
					dist += l2;
					++hops;
				}
				if (hops < 8) cls = hops <= 1 ? 1u : hops <= 2 ? 2u : hops <= 4 ? 3u : hops <= 6 ? 4u : 5u;
				else {
					uint32_t est = (8u * (uint32_t)kMaxDist) / dist; // candidates if the chain stays this dense
					if (est > chain) est = chain;
					cls = est <= 11 ? 6u : est <= 16 ? 7u : est <= 23 ? 8u : est <= 32 ? 9u : est <= 45 ? 10u : est <= 64 ? 11u
					      : est <= 91 ? 12u : est <= 128 ? 13u : est <= 512 ? 14u : 15u;
				}
			}
		}
		const uint32_t peers = __match_any_sync(0xffffffffu, cls);
		if (cls && lane == __ffs((int)peers) - 1) atomicAdd(&s_cls[0][cls], (uint32_t)__popc(peers));
		cw[k >> 3] |= cls << ((k & 7) * 4);
	}
	__syncthreads();
	uint32_t total = 0;
	{
		// class bases, longest walks first
		uint32_t b = 0;
		uint32_t mine = 0;
		for (int c = kMatchClasses - 1; c >= 1; c--) {
			if ((int)threadIdx.x == c) mine = b;
			b += s_cls[0][c];
		}
		total = b;
		__syncthreads();
		if (threadIdx.x >= 1 && threadIdx.x < kMatchClasses) s_cls[1][threadIdx.x] = mine;
		__syncthreads();
	}
#pragma unroll
	for (int k = 0; k < kTile / kMatchThreads; k++) {
		const uint32_t cls = (cw[k >> 3] >> ((k & 7) * 4)) & 15u;
		const uint32_t peers = __match_any_sync(0xffffffffu, cls);
		uint32_t slot = 0;
		const int leader = __ffs((int)peers) - 1;
		if (cls && lane == leader) slot = atomicAdd(&s_cls[1][cls], (uint32_t)__popc(peers));
		slot = __shfl_sync(0xffffffffu, slot, leader);
		if (cls) order[slot + (uint32_t)__popc(peers & ((1u << lane) - 1u))] = (uint16_t)(threadIdx.x + (uint32_t)k * kMatchThreads);
	}
	__syncthreads();
	for (uint32_t i = threadIdx.x; i < total; i += kMatchThreads) {
		const uint32_t p = t0 + (uint32_t)__ldcg(&order[i]);
		const uint32_t la = n - p;
		const uint32_t maxlen = la < (uint32_t)kMaxMatch ? la : (uint32_t)kMaxMatch;
		const uint32_t nice = la < (uint32_t)lp.nice ? la : (uint32_t)lp.nice;
		const int is = (int)(p - w0);
		const uint8_t *sp = s_data + is;
		// The walk runs on window indices, offset by m so that the hot loop addresses the candidate's byte m directly:
		// icm = candidate + m, lom = lo + m with lo the lowest index a later chain member may have (distance < 32506, T7),
		// lk = the link window shifted by -m.  The re-encoded chain end lands below lo as well, so one compare per hop
		// ends the walk.  A listed position always has a first candidate (see above).
		uint32_t m = kMinMatch - 1, bd = 0, resB = 0;
		int icm = is - (int)s_link[is] + (int)m;
		int lom = is - (kMaxDist - 1) + (int)m;
		const uint16_t *lk = s_link - m;
		bool haveB = false;
		uint32_t stop = budgetB ? budgetB : chain;
		uint32_t left = stop; // candidates to test before the next budget event
		const uint32_t s0 = sp[0], s1 = sp[1];
		uint32_t scan_end1 = s1, scan_end = sp[2];
		// bytes 2..9 of the scan string stay in registers: most extensions end inside them
		uint32_t sw0, sw1;
		{
			const uint32_t as = (uint32_t)is + 2;
			const uint32_t *ws = reinterpret_cast<const uint32_t *>(s_data + (as & ~3u));
			const uint32_t w1 = ws[1], sh = (as & 3u) * 8u;
			sw0 = __funnelshift_r(ws[0], w1, sh);
			sw1 = __funnelshift_r(w1, ws[2], sh);
		}
		// Every level 5-9 budget (chain and chain >> 2) is a multiple of four: the walk steps four candidates per budget
		// test (b200z_core.cuh asserts it).  The lanes of a warp step their candidates together; only a candidate whose
		// byte m matches leaves the straight path.  (Tried and dropped: the rejects in a loop of their own, without the
		// convergence region around the rare path -- fewer instructions, but the lanes no longer step together: DESIGN.md §7b.)
		for (;;) {
#pragma unroll
			for (int j = 0; j < 4; j++) {
				const uint32_t b = s_data[icm];
				int nx = icm - (int)lk[icm];
				if (b == scan_end) {
					const int ic = icm - (int)m;
					const uint8_t *c = s_data + ic;
					// the other three bytes of the quick test in one branch: their loads are issued together
					if ((c[m - 1] == scan_end1) & (c[0] == s0) & (c[1] == s1)) {
						uint32_t l = 2;
						if (maxlen >= 10) {
							const uint32_t ac = (uint32_t)ic + 2;
							const uint32_t *wc = reinterpret_cast<const uint32_t *>(s_data + (ac & ~3u));
							const uint32_t w1 = wc[1], sh = (ac & 3u) * 8u;
							uint32_t x = __funnelshift_r(wc[0], w1, sh) ^ sw0;
							if (x) {
								l = 2 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
								goto lcp_done;
							}
							x = __funnelshift_r(w1, wc[2], sh) ^ sw1;
							if (x) {
								l = 6 + ((uint32_t)(__ffs((int)x) - 1) >> 3);
								goto lcp_done;
							}
							l = 10;
						}
						while (l + 4 <= maxlen) {
							const uint32_t ac = (uint32_t)ic + l, as = (uint32_t)is + l;
							const uint32_t *wc = reinterpret_cast<const uint32_t *>(s_data + (ac & ~3u));
							const uint32_t *ws = reinterpret_cast<const uint32_t *>(s_data + (as & ~3u));
							const uint32_t x = __funnelshift_r(wc[0], wc[1], (ac & 3u) * 8u) ^ __funnelshift_r(ws[0], ws[1], (as & 3u) * 8u);
							if (x) {
								l += (uint32_t)(__ffs((int)x) - 1) >> 3;
								goto lcp_done;
							}
							l += 4;
						}
						while (l < maxlen && c[l] == sp[l]) ++l;
					lcp_done:
						if (l > m) {
							bd = (uint32_t)(is - ic);
							if (l >= nice) {
								m = l;
								goto done;
							}
							nx += (int)(l - m);
							lom += (int)(l - m);
							lk -= l - m;
							m = l;
							scan_end1 = sp[m - 1];
							scan_end = sp[m];
						}
					}
				}
				icm = nx;
				if (icm < lom) goto done;
			}
			left -= 4;
			if (left == 0) { // first the quarter budget (B's snapshot), then the full one
				if (stop == chain) break;
				resB = m >= (uint32_t)kMinMatch ? pack_match(m, bd) : 0u;
				haveB = true;
				left = chain - stop;
				stop = chain;
			}
		}
	done:
		const uint32_t resA = m >= (uint32_t)kMinMatch ? pack_match(m, bd) : 0u;
		out[p] = make_uint2(resA, haveB ? resB : resA);
	}
}

// ------------------------------------------------------------------------------------------------
// K3: the lazy parse (DeflateSlow's state machine, DeflaterEngine.cs:741-855), parallel at three levels.
//
//  lanes   : a ROUND is 32 segments x kSeg positions.  The round's table entries and bytes are staged in shared memory
//            (cp.async), every lane parses its own segment starting from a guessed clean state, then each lane hands
//            its exit state to the next lane as that lane's entry; lanes whose entry changed parse again.  Lane 0's
//            entry is the true carried state, so after k hand-offs the first k+1 lanes are exact; because the parse
//            re-synchronises within a few symbols the hand-offs normally stop changing anything after one iteration.
//            A final pass emits the round's symbols into the round's own slot.
//  chunks  : k_parse_chunk runs one warp per CHUNK of a stream (many chunks per stream, all concurrent), every chunk
//            but the first starting from a guessed clean state; per round it records the exit state and symbol count.
//  fix-up  : k_parse_fix walks the chunks of a stream in order and re-runs rounds of a chunk from the true entry state
//            until a round's exit state equals the recorded one -- from there on the speculative result stands.
//  gather  : k_parse_scan prefix-sums the rounds' symbol counts, k_parse_gather moves the symbols to their final
//            positions and records the block cuts (every 16384 symbols, DeflaterHuffman.cs:863).
// ------------------------------------------------------------------------------------------------
constexpr int kSegShift = 5;
constexpr int kSeg = 1 << kSegShift; // 32 positions per lane: 9.6 KiB of shared memory per warp, 22 warps per SM
constexpr int kRound = 32 * kSeg;
constexpr int kParseWarm = 128; // positions a chunk parses in front of its first one to find its entry state (k_parse_chunk)
constexpr int kSegStride = kSeg + 2; // uint2 entries; +2 keeps 16-byte alignment for cp.async and staggers the banks
constexpr int kParseDatOff = 32 * kSegStride * 8;
constexpr int kParseSmem = kParseDatOff + kRound + 48;

struct ChunkDesc {
	int32_t stream;
	uint32_t c0, c1; // positions [c0, c1) of the stream, c0 a multiple of kRound
};

__device__ __forceinline__ ParseCarry shfl_carry(const ParseCarry &c, int src) {
	ParseCarry r;
	r.st.p = __shfl_sync(0xffffffffu, c.st.p, src);
	r.st.mlen = __shfl_sync(0xffffffffu, c.st.mlen, src);
	r.st.mstart = __shfl_sync(0xffffffffu, c.st.mstart, src);
	r.st.prevAvail = __shfl_sync(0xffffffffu, c.st.prevAvail, src);
	r.last_top = __shfl_sync(0xffffffffu, c.last_top, src);
	return r;
}

__device__ __forceinline__ ParseCarry clean_carry(uint32_t p) {
	ParseCarry c;
	parse_init(c.st);
	c.st.p = p;
	c.last_top = p;
	return c;
}

struct RoundRec { // what a round leaves behind (5 + 1 words)
	uint32_t p, mlen, mstart, prevAvail, last_top, cnt;
};
// The first loop top a run does not parse.  Finish / Flush parse to the end; an open run (B200Z_END_NONE) stops where
// DeflateSlow's BUSY_STATE loop stops, at the first loop top with less than MIN_LOOKAHEAD bytes ahead (a match taken at an
// earlier one may still reach beyond it).  Every top in front of it sees at least 262 bytes, so its match table entries
// and its step are the same as in a run over more input.
__device__ __forceinline__ uint32_t parse_end(uint32_t n, int end_mode) {
	constexpr uint32_t kMinLookahead = kMaxMatch + kMinMatch + 1;
	if (end_mode != B200Z_END_NONE) return n;
	return n >= kMinLookahead ? n - (kMinLookahead - 1) : 0u;
}
__device__ __forceinline__ ParseCarry rec_carry(const RoundRec &r) {
	ParseCarry c;
	c.st.p = r.p;
	c.st.mlen = r.mlen;
	c.st.mstart = r.mstart;
	c.st.prevAvail = r.prevAvail;
	c.last_top = r.last_top;
	return c;
}

// One round [base, base + kRound) of a stream, entered with `carry` (uniform across the warp; updated to the round's
// exit state).  Loop tops at or behind `pend` are left alone (parse_end).  The round's symbols go to sround[0 .. cnt).
// Returns cnt (uniform).
__device__ __forceinline__ uint32_t parse_round(uint8_t *smem, const uint8_t *data, const uint16_t *lnk, const uint2 *tab,
                                                uint32_t n, uint32_t pend, uint32_t H, uint32_t ab, uint32_t base,
                                                const LevelParams &lp, int strategy, ParseCarry &carry, uint32_t *sround) {
	uint2 *s_tab = reinterpret_cast<uint2 *>(smem);
	uint8_t *s_dat = smem + kParseDatOff; // s_dat[16 + i] = byte at position base + i (16 bytes of history in front)
	const int lane = threadIdx.x & 31;
	const uint32_t rn = (n - base > (uint32_t)kRound) ? (uint32_t)kRound : n - base;
	__syncwarp();
	// stage the round with 16-byte async copies (LDGSTS): all of them are in flight at once, no register staging
	for (uint32_t i = 2 * lane; i + 1 < rn; i += 64)
		__pipeline_memcpy_async(&s_tab[(i >> kSegShift) * kSegStride + (i & (kSeg - 1))], &tab[base + i], 16);
	{
		// bytes [base - 16, base + rn) rounded up to 16 (the input slot has 16 bytes of slack behind n)
		const uint32_t c0 = base ? 0u : 1u, c1 = (16 + rn + 15) >> 4;
		for (uint32_t c = c0 + lane; c < c1; c += 32) __pipeline_memcpy_async(s_dat + 16 * c, data + base - 16 + 16 * c, 16);
	}
	__pipeline_commit();
	if ((rn & 1) && lane == 0) s_tab[((rn - 1) >> kSegShift) * kSegStride + ((rn - 1) & (kSeg - 1))] = tab[base + rn - 1];
	__pipeline_wait_prior(0);
	__syncwarp();
	const uint32_t seg_end = base + (uint32_t)(lane + 1) * kSeg;
	auto tabf = [&](uint32_t p, uint32_t &a, uint32_t &b) {
		const uint32_t i = p - base;
		const uint2 t = s_tab[(i >> kSegShift) * kSegStride + (i & (kSeg - 1))];
		a = t.x;
		b = t.y;
	};
	auto bytef = [&](uint32_t q) { return (uint32_t)s_dat[q + 16 - base]; };
	auto slowf = [&](uint32_t p, uint32_t m0, uint32_t budget) { return match_search_above(data, lnk, p, n, m0, budget, ab); };
	ParseCarry entry, ex;
	if (lane == 0) entry = carry;
	else {
		const uint32_t ss = base + (uint32_t)lane * kSeg;
		entry = clean_carry(ss > H ? ss : H); // history positions are never parsed; the state at H is exactly "clean"
	}
	ex = entry;
	uint32_t cnt = 0;
	bool changed = true;
	const uint32_t lim = seg_end < pend ? seg_end : pend;
	for (int it = 0; it < 34; it++) {
		// all lanes step together and re-converge every iteration (a per-lane loop would leave them diverged)
		if (changed) {
			ex = entry;
			cnt = 0;
		}
		bool act = changed && ex.st.p < lim;
		while (__any_sync(0xffffffffu, act)) {
			if (act) {
				ex.last_top = ex.st.p;
				uint32_t s2;
				cnt += (uint32_t)parse_step(ex.st, n, lp, strategy, tabf, bytef, slowf, s2);
				act = ex.st.p < lim;
			}
			__syncwarp();
		}
		const ParseCarry ne = shfl_carry(ex, lane == 0 ? 0 : lane - 1);
		changed = false;
		if (lane > 0) {
			changed = !carry_equal(ne, entry);
			entry = ne;
		}
		if (!__any_sync(0xffffffffu, changed)) break;
	}
	// final pass: emit at prefix-summed offsets inside the round's slot
	uint32_t incl = cnt;
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
		if (lane >= o) incl += t;
	}
	uint32_t idx = incl - cnt;
	ParseCarry c = entry;
	{
		bool act = c.st.p < lim;
		while (__any_sync(0xffffffffu, act)) {
			if (act) {
				c.last_top = c.st.p;
				uint32_t s2;
				if (parse_step(c.st, n, lp, strategy, tabf, bytef, slowf, s2)) sround[idx++] = s2;
				act = c.st.p < lim;
			}
			__syncwarp();
		}
	}
	carry = shfl_carry(c, 31);
	return __shfl_sync(0xffffffffu, incl, 31);
}

__global__ void __launch_bounds__(32)
    k_parse_chunk(const uint8_t *__restrict__ in, const uint16_t *__restrict__ link, const uint2 *__restrict__ mt,
                  uint32_t *__restrict__ sym_local, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                  const ChunkDesc *__restrict__ chunks, const uint32_t *__restrict__ rnd_off, RoundRec *__restrict__ recs,
                  RoundRec *__restrict__ ents, const uint32_t *__restrict__ hist, const int64_t *__restrict__ bias,
                  const RoundRec *__restrict__ entry, LevelParams lp, int strategy, int warm, int end_mode) {
	extern __shared__ __align__(16) uint8_t smem[];
	const ChunkDesc cd = chunks[blockIdx.x];
	const uint32_t n = (uint32_t)in_len[cd.stream];
	const uint32_t pend = parse_end(n, end_mode);
	const int64_t off = in_off[cd.stream];
	RoundRec *rr = recs + rnd_off[cd.stream];
	const uint32_t H = hist[cd.stream], ab = (uint32_t)bias[cd.stream];
	// exact for the first chunk: the stream's entry state (DeflaterEngine.Reset :234-253, the state right after a dictionary
	// or a flush, or what an open run left at its cut).  Every other chunk parses kParseWarm positions in front of its first
	// one from a clean state (lane 0, straight from global memory): DeflateSlow's state re-synchronises within a few symbols,
	// so the state this reaches at c0 is the true one at 99.8 % of the boundaries (tools/tile_fixup.cpp).  It is recorded;
	// k_parse_fix compares it with the exit of the chunk in front and parses again only where they differ.
	ParseCarry carry = cd.c0 == 0 ? rec_carry(entry[cd.stream]) : clean_carry(cd.c0 > H ? cd.c0 : H);
	if (cd.c0 > H && warm > 0) {
		if (threadIdx.x == 0) {
			const uint8_t *data = in + off;
			const uint16_t *lnk = link + off;
			const uint2 *tab = mt + off;
			const uint32_t ws = cd.c0 - H > (uint32_t)warm ? cd.c0 - (uint32_t)warm : H;
			ParseCarry w = clean_carry(ws);
			auto tabg = [&](uint32_t p, uint32_t &a, uint32_t &b) {
				const uint2 t = tab[p];
				a = t.x;
				b = t.y;
			};
			auto byteg = [&](uint32_t q) { return (uint32_t)data[q]; };
			auto slowg = [&](uint32_t p, uint32_t m0, uint32_t budget) { return match_search_above(data, lnk, p, n, m0, budget, ab); };
			while (w.st.p < cd.c0) {
				w.last_top = w.st.p;
				uint32_t s2;
				parse_step(w.st, n, lp, strategy, tabg, byteg, slowg, s2);
			}
			carry = w;
		}
		carry = shfl_carry(carry, 0);
	}
	if (threadIdx.x == 0) {
		RoundRec e;
		e.p = carry.st.p;
		e.mlen = carry.st.mlen;
		e.mstart = carry.st.mstart;
		e.prevAvail = carry.st.prevAvail;
		e.last_top = carry.last_top;
		e.cnt = 0;
		ents[rnd_off[cd.stream] + cd.c0 / kRound] = e;
	}
	for (uint32_t base = cd.c0; base < cd.c1; base += kRound) {
		const uint32_t cnt = parse_round(smem, in + off, link + off, mt + off, n, pend, H, ab, base, lp, strategy, carry, sym_local + off + base);
		if (threadIdx.x == 0) {
			RoundRec r;
			r.p = carry.st.p;
			r.mlen = carry.st.mlen;
			r.mstart = carry.st.mstart;
			r.prevAvail = carry.st.prevAvail;
			r.last_top = carry.last_top;
			r.cnt = cnt;
			rr[base / kRound] = r;
		}
	}
}

__global__ void __launch_bounds__(32)
    k_parse_fix(const uint8_t *__restrict__ in, const uint16_t *__restrict__ link, const uint2 *__restrict__ mt,
                uint32_t *__restrict__ sym_local, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                const uint32_t *__restrict__ rnd_off, RoundRec *__restrict__ recs, const RoundRec *__restrict__ ents, uint32_t chunk,
                const uint32_t *__restrict__ hist, const int64_t *__restrict__ bias, LevelParams lp, int strategy, int end_mode) {
	extern __shared__ __align__(16) uint8_t smem[];
	const int stream = blockIdx.x;
	const uint32_t n = (uint32_t)in_len[stream];
	const uint32_t pend = parse_end(n, end_mode);
	if (n <= chunk) return; // a single chunk was parsed from the true initial state
	const int64_t off = in_off[stream];
	RoundRec *rr = recs + rnd_off[stream];
	const RoundRec *en = ents + rnd_off[stream];
	const uint32_t H = hist[stream], ab = (uint32_t)bias[stream];
	const uint32_t nchunks = (n + chunk - 1) / chunk;
	const int lane = threadIdx.x;
	// Boundaries are checked 32 at a time: the entry a chunk used against the exit of the chunk in front (exact by induction
	// once every boundary before it has been checked).  The first that differs is parsed again from the true state until a
	// round's exit equals the recorded one; the scan then goes on behind it (its own exit may have changed).
	uint32_t k0 = 1;
	while (k0 < nchunks) {
		const uint32_t k = k0 + (uint32_t)lane;
		bool bad = false;
		if (k < nchunks) {
			const uint32_t c0 = k * chunk;
			const ParseCarry truth = rec_carry(rr[c0 / kRound - 1]);
			ParseCarry used = rec_carry(en[c0 / kRound]);
			used.last_top = truth.last_top; // irrelevant here: the chunk processes at least one loop top
			bad = !carry_equal(truth, used);
		}
		const uint32_t mask = __ballot_sync(0xffffffffu, bad);
		if (!mask) {
			k0 += 32;
			continue;
		}
		const uint32_t kk = k0 + (uint32_t)(__ffs((int)mask) - 1);
		const uint32_t c0 = kk * chunk;
		const uint32_t c1 = (n - c0 > chunk) ? c0 + chunk : n;
		ParseCarry truth = rec_carry(rr[c0 / kRound - 1]);
		for (uint32_t base = c0; base < c1; base += kRound) {
			const ParseCarry old_exit = rec_carry(rr[base / kRound]);
			const uint32_t cnt = parse_round(smem, in + off, link + off, mt + off, n, pend, H, ab, base, lp, strategy, truth,
			                                 sym_local + off + base);
			__syncwarp();
			if (lane == 0) {
				RoundRec r;
				r.p = truth.st.p;
				r.mlen = truth.st.mlen;
				r.mstart = truth.st.mstart;
				r.prevAvail = truth.st.prevAvail;
				r.last_top = truth.last_top;
				r.cnt = cnt;
				rr[base / kRound] = r;
			}
			__syncwarp();
			if (carry_equal(truth, old_exit)) break; // re-synchronised: the rest of the chunk stands as parsed
		}
		__syncwarp();
		k0 = kk + 1;
	}
}

// exclusive scan of the rounds' symbol counts of one stream; also the end-of-stream bookkeeping
__global__ void __launch_bounds__(256)
    k_parse_scan(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                 const uint32_t *__restrict__ rnd_off, const RoundRec *__restrict__ recs, uint32_t *__restrict__ rnd_symoff,
                 uint32_t *__restrict__ sym, uint32_t *__restrict__ nsyms, uint32_t *__restrict__ nblocks,
                 const uint32_t *__restrict__ blk_off, uint32_t *__restrict__ blk_start, uint32_t *__restrict__ blk_ptop,
                 const uint32_t *__restrict__ hist, int end_mode) {
	__shared__ uint32_t s_part[8];
	__shared__ uint32_t s_carry;
	const int stream = blockIdx.x;
	const uint32_t n = (uint32_t)in_len[stream];
	const uint32_t nr = (n + kRound - 1) / kRound;
	const RoundRec *rr = recs + rnd_off[stream];
	uint32_t *so = rnd_symoff + rnd_off[stream];
	if (threadIdx.x == 0) s_carry = 0;
	__syncthreads();
	for (uint32_t b = 0; b < nr; b += 256) {
		const uint32_t i = b + threadIdx.x;
		const uint32_t v = i < nr ? rr[i].cnt : 0u;
		uint32_t incl = v;
		for (int o = 1; o < 32; o <<= 1) {
			const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if ((threadIdx.x & 31) >= o) incl += t;
		}
		if ((threadIdx.x & 31) == 31) s_part[threadIdx.x >> 5] = incl;
		__syncthreads();
		uint32_t woff = 0;
		for (int k = 0; k < (int)(threadIdx.x >> 5); k++) woff += s_part[k];
		const uint32_t carry = s_carry;
		if (i < nr) so[i] = carry + woff + incl - v;
		__syncthreads();
		if (threadIdx.x == 255) s_carry = carry + woff + incl;
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		uint32_t total = s_carry;
		const uint32_t H = hist[stream];
		ParseCarry fin = nr ? rec_carry(rr[nr - 1]) : clean_carry(H);
		uint32_t *bstart = blk_start + blk_off[stream];
		uint32_t *bptop = blk_ptop + blk_off[stream];
		bstart[0] = H;
		uint32_t nblk = total >> 14;
		const bool ended_full = end_mode == B200Z_END_FINISH && total > 0 && (total & (uint32_t)(kBlockSyms - 1)) == 0 && !fin.st.prevAvail;
		// an open run writes the blocks the symbol rule closed and nothing else: the rest is parsed again by the next run
		if (!ended_full && end_mode != B200Z_END_NONE) {
			// final flush at lookahead == 0 (DeflaterEngine.cs:750-768)
			if (fin.st.prevAvail) (sym + in_off[stream])[total++] = sym_lit(in[in_off[stream] + fin.st.p - 1]);
			bptop[nblk] = fin.last_top;
			++nblk;
		}
		nsyms[stream] = total;
		nblocks[stream] = nblk;
	}
}

// moves every round's symbols to their final place and records the block cuts that fall inside the round
__global__ void __launch_bounds__(128)
    k_parse_gather(const uint32_t *__restrict__ sym_local, uint32_t *__restrict__ sym, const int64_t *__restrict__ in_off,
                   const int64_t *__restrict__ in_len, const int2 *__restrict__ rnd_desc, const uint32_t *__restrict__ rnd_off,
                   const RoundRec *__restrict__ recs, const uint32_t *__restrict__ rnd_symoff, const uint32_t *__restrict__ blk_off,
                   uint32_t *__restrict__ blk_start, uint32_t *__restrict__ blk_ptop, const uint32_t *__restrict__ hist) {
	const int2 d = rnd_desc[blockIdx.x]; // (stream, first round of this CTA's group of 4)
	const int64_t off = in_off[d.x];
	const uint32_t n = (uint32_t)in_len[d.x];
	const uint32_t nr = (n + kRound - 1) / kRound;
	const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const uint32_t r = (uint32_t)d.y + (uint32_t)w;
	if (r >= nr) return;
	const RoundRec *rr = recs + rnd_off[d.x];
	const uint32_t cnt = rr[r].cnt;
	const uint32_t dst0 = rnd_symoff[rnd_off[d.x] + r];
	const uint32_t *src = sym_local + off + r * (uint32_t)kRound;
	uint32_t *dst = sym + off + dst0;
	for (uint32_t i = lane; i < cnt; i += 32) dst[i] = src[i];
	// block cuts: global symbol index idx with (idx + 1) % 16384 == 0
	if (lane == 0 && cnt) {
		const uint32_t first_b = (dst0 + (uint32_t)kBlockSyms) >> 14;          // smallest b with b * 16384 - 1 >= dst0
		const uint32_t last_idx = dst0 + cnt - 1;
		if (first_b * (uint32_t)kBlockSyms - 1 <= last_idx) {
			// bytes covered before this round's first symbol: entry.p, minus the pending literal if there is one
			uint32_t bytes;
			if (r == 0) bytes = hist[d.x];
			else bytes = rr[r - 1].p - (rr[r - 1].prevAvail ? 1u : 0u);
			uint32_t *bstart = blk_start + blk_off[d.x];
			uint32_t *bptop = blk_ptop + blk_off[d.x];
			uint32_t nextb = first_b;
			for (uint32_t i = 0; i < cnt; i++) {
				const uint32_t s2 = src[i];
				const uint32_t L = sym_len(s2);
				bytes += L;
				if (dst0 + i + 1 == nextb * (uint32_t)kBlockSyms) {
					// the loop top at which the symbol was tallied: literal -> the position after it; match -> its start + 1
					bptop[nextb - 1] = sym_dist(s2) ? bytes - L + 1 : bytes;
					bstart[nextb] = bytes;
					++nextb;
				}
			}
		}
	}
}

// Open runs (B200Z_END_NONE): the parse state right behind the last block cut, i.e. behind the tally of symbol K - 1 with
// K = nblocks * 16384, which the next run of the stream is entered with (its byte `p - prevAvail` is the first one not
// written).  The rounds only record their exit states, so the round holding symbol K - 1 is parsed again from its entry up
// to the cut: at most one round of loop tops, one thread per stream.  Without a cut the entry stands.
__global__ void k_parse_cut(const uint8_t *__restrict__ in, const uint16_t *__restrict__ link, const uint2 *__restrict__ mt,
                            const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len, const uint32_t *__restrict__ rnd_off,
                            const RoundRec *__restrict__ recs, const uint32_t *__restrict__ rnd_symoff,
                            const uint32_t *__restrict__ nblocks, const int64_t *__restrict__ bias, const RoundRec *__restrict__ entry,
                            RoundRec *__restrict__ cut, int nstreams, LevelParams lp, int strategy) {
	const int stream = blockIdx.x * blockDim.x + threadIdx.x;
	if (stream >= nstreams) return;
	const uint32_t n = (uint32_t)in_len[stream];
	const uint32_t K = nblocks[stream] * (uint32_t)kBlockSyms;
	ParseCarry c = rec_carry(entry[stream]);
	if (K > 0) {
		const int64_t off = in_off[stream];
		const uint8_t *data = in + off;
		const uint16_t *lnk = link + off;
		const uint2 *tab = mt + off;
		const uint32_t ab = (uint32_t)bias[stream];
		const uint32_t *so = rnd_symoff + rnd_off[stream];
		const RoundRec *rr = recs + rnd_off[stream];
		// the last round whose first symbol comes before K holds symbol K - 1 (symbol offsets never decrease)
		uint32_t lo = 0, hi = (n + kRound - 1) / kRound - 1;
		while (lo < hi) {
			const uint32_t mid = (lo + hi + 1) >> 1;
			if (so[mid] < K) lo = mid;
			else hi = mid - 1;
		}
		if (lo > 0) c = rec_carry(rr[lo - 1]);
		auto tabg = [&](uint32_t p, uint32_t &a, uint32_t &b) {
			const uint2 t = tab[p];
			a = t.x;
			b = t.y;
		};
		auto byteg = [&](uint32_t q) { return (uint32_t)data[q]; };
		auto slowg = [&](uint32_t p, uint32_t m0, uint32_t budget) { return match_search_above(data, lnk, p, n, m0, budget, ab); };
		for (uint32_t k = so[lo]; k < K;) {
			c.last_top = c.st.p;
			uint32_t s2;
			k += (uint32_t)parse_step(c.st, n, lp, strategy, tabg, byteg, slowg, s2);
		}
	}
	RoundRec r;
	r.p = c.st.p;
	r.mlen = c.st.mlen;
	r.mstart = c.st.mstart;
	r.prevAvail = c.st.prevAvail;
	r.last_top = c.last_top;
	r.cnt = K;
	cut[stream] = r;
}

// ------------------------------------------------------------------------------------------------
// Levels 1-4: DeflateFast.  The chains depend on the parse, so a stream is parsed serially by lane 0 with the
// reference's own head[]/prev[] tables (shared memory, 128 KiB); SlideWindow's table sweep is done by the whole warp.
// All streams of the batch run concurrently (one warp each).  Symbols and block cuts feed k_plan / k_scan / k_emit.
// ------------------------------------------------------------------------------------------------
constexpr int kFastSmem = 2 * 32768 * 2; // prev[] (+ head[] when a batch has no more streams than the GPU has SMs)

// eight window bytes starting at slot byte `a`, first byte in the low bits of lo (aligned words; the slot is 256-byte
// aligned and has 16 bytes of slack behind its data)
__device__ __forceinline__ void fast_load8(const uint8_t *__restrict__ in, uint32_t a, uint32_t &lo, uint32_t &hi) {
	const uint32_t *p = reinterpret_cast<const uint32_t *>(in + (a & ~3u));
	const uint32_t w0 = p[0], w1 = p[1], w2 = p[2];
	const uint32_t sh = (a & 3u) * 8u;
	lo = __funnelshift_r(w0, w1, sh);
	hi = __funnelshift_r(w1, w2, sh);
}

// The warp-wide group step of DeflateFast (DeflaterEngine.cs:651-739), `nl` consecutive loop tops at once.
//
// What makes DeflateFast serial is that a match longer than max_lazy leaves its inner positions out of the hash chains
// (:699-715); a literal or a match of at most max_lazy bytes inserts every position it covers.  So as long as no long match
// is taken, "every position of the group is a chain member" is the truth, and the searches of all loop tops can run at once:
// lane j takes window index s0 + j, its chain head is the nearest lower lane with the same hash (else head[]), links of
// group positions are written to prev[] up front (slots of positions further back than MAX_DIST are never read again), every
// lane runs FindLongestMatch from matchLen = 2 with the level's chain budget and remembers which group positions it
// tested (`used`).  The parse is replayed over the lanes' results in order by a cursor v that all lanes keep: a lane is
// resolved once its walk is complete; a long match at lane v takes positions v+1 .. v+len-1 out (set N) and ends their
// walks; a later lane whose walk touched N is not trusted -- the group ends in front of it and the next step starts there.
// Lanes behind a long match that never touched N saw exactly the chains the reference sees (a walk that read a link into N
// either tested that position -- then it is in `used` -- or had run out of budget).  At commit the links of the inserted
// positions are recomputed over the inserted lanes only, head[] gets the last inserted position of every hash, the visited
// lanes write their symbols in order.
//
// Latency is what this kernel pays for, so: a lane gathers up to four chain members before it loads any of them (one
// memory round trip per four candidates); a candidate that still matches after 16 bytes waits until its lane is the
// cursor and is then extended by the whole warp (8 bytes per lane) -- lanes inside a long repeat never get there, the match
// of the lane in front of them covers them first.
//
// s0 / la / nsym / total: the engine's strstart, lookahead, symbols in the block, symbols written (uniform over the warp; the
// caller keeps lane 0's FastEngine in step).  Returns 1 if the last action was a long match (UpdateHash is due, :712-714).
__device__ __forceinline__ int fast_lcp8(uint32_t alo, uint32_t ahi, uint32_t blo, uint32_t bhi) {
	uint32_t x = alo ^ blo;
	if (x) return (__ffs((int)x) - 1) >> 3;
	x = ahi ^ bhi;
	if (x) return 4 + ((__ffs((int)x) - 1) >> 3);
	return 8;
}

__device__ __forceinline__ int fast_group_step(const uint8_t *__restrict__ in, uint32_t woff, uint16_t *head, uint16_t *prev,
                                               const LevelParams &lp, int lane, int nl, int &s0, int &la, uint32_t &nsym,
                                               uint32_t *__restrict__ sout, uint32_t &total, int &last_h, int &match_start) {
	const uint32_t full = 0xffffffffu;
	const uint32_t lt = (1u << lane) - 1u;
	const int q = s0 + lane;
	const uint32_t qa = (uint32_t)q + woff;
	const bool active = lane < nl;
	uint32_t lo, hi;
	fast_load8(in, qa, lo, hi);
#if !defined(B200Z_EMU)
	// the bytes a later step starts from: one 128-byte line per lane pair, 2 KiB ahead (reads past the slot stay inside the
	// plan's input blob or its tail padding; a prefetch does not fault)
	if (la > 4096 && (lane & 1)) asm volatile("prefetch.global.L2 [%0];" ::"l"(in + ((qa + 2048u + 64u * (uint32_t)lane) & ~127u)));
#endif
	const uint32_t h = hash3(lo & 255u, (lo >> 8) & 255u, (lo >> 16) & 255u);
	const int hh = head[h];
	const uint32_t same = __match_any_sync(full, active ? h : (0x8000u | (uint32_t)lane));
	const uint32_t pm = same & lt;
	const int cand0 = pm ? s0 + (31 - __clz((int)pm)) : hh;
	if (active) prev[q & 32767] = (uint16_t)cand0;
	__syncwarp();

	// FindLongestMatch (:474-612) from matchLen = MIN_MATCH - 1: the longest common prefix with every chain member in chain
	// order, the first longest wins, stop at nice_length; the reference's scan_end tests only skip members that cannot win
	int best = kMinMatch - 1, bestc = 0, chain = lp.chain;
	uint32_t used = 0;
	const int limit = q - kMaxDist > 0 ? q - kMaxDist : 0;
	int cand = (active && cand0 != 0 && q - cand0 <= kMaxDist) ? cand0 : 0; // next chain member to gather (0: none left)
	bool go = cand != 0;    // the walk is not complete
	bool pend = false;      // the member at bi matches for >= 16 bytes and waits for the warp
	int c0 = 0, c1 = 0, c2 = 0, c3 = 0, nb = 0, bi = 0;
	uint32_t l0 = 0, h0 = 0, l1 = 0, h1 = 0, l2 = 0, h2 = 0, l3 = 0, h3 = 0;
	uint32_t visited = 0, N = 0;
	int v = 0, last_long = 0;
	bool stop = false;
	for (;;) {
		if (go && bi == nb) {
			// the next (up to) four members: `do test while ((cur = prev[cur]) > limit && --chain)`
			nb = 0;
			bi = 0;
#define B200Z_GATHER(C)                                                                                                           \
	if (cand) {                                                                                                                    \
		C = cand;                                                                                                                   \
		++nb;                                                                                                                       \
		const int nx = prev[cand & 32767];                                                                                          \
		cand = (nx > limit && --chain != 0) ? nx : 0;                                                                               \
	}
			B200Z_GATHER(c0)
			B200Z_GATHER(c1)
			B200Z_GATHER(c2)
			B200Z_GATHER(c3)
#undef B200Z_GATHER
			if (nb > 0) fast_load8(in, (uint32_t)c0 + woff, l0, h0);
			if (nb > 1) fast_load8(in, (uint32_t)c1 + woff, l1, h1);
			if (nb > 2) fast_load8(in, (uint32_t)c2 + woff, l2, h2);
			if (nb > 3) fast_load8(in, (uint32_t)c3 + woff, l3, h3);
			if (nb == 0) go = false;
		}
#define B200Z_TEST(K, C, CL, CH)                                                                                                 \
	if (go && !pend && bi == K && K < nb) {                                                                                        \
		if (C >= s0) used |= 1u << (C - s0);                                                                                        \
		int l = fast_lcp8(CL, CH, lo, hi);                                                                                          \
		if (l == 8) {                                                                                                               \
			uint32_t a0, a1, b0, b1;                                                                                                 \
			fast_load8(in, (uint32_t)C + woff + 8u, a0, a1);                                                                         \
			fast_load8(in, qa + 8u, b0, b1);                                                                                         \
			l += fast_lcp8(a0, a1, b0, b1);                                                                                          \
		}                                                                                                                           \
		if (l == 16) {                                                                                                              \
			pend = true;                                                                                                             \
		} else {                                                                                                                    \
			if (l > best) {                                                                                                          \
				best = l;                                                                                                             \
				bestc = C;                                                                                                            \
				if (best >= lp.nice) go = false;                                                                                      \
			}                                                                                                                        \
			bi = K + 1;                                                                                                              \
		}                                                                                                                           \
	}
		B200Z_TEST(0, c0, l0, h0)
		B200Z_TEST(1, c1, l1, h1)
		B200Z_TEST(2, c2, l2, h2)
		B200Z_TEST(3, c3, l3, h3)
#undef B200Z_TEST
		if (go && !pend && bi == nb && cand == 0) go = false; // every member tested
		// the cursor's lane is extended by the warp: lane k compares bytes 16 + 8k .. 16 + 8k + 7 (MAX_MATCH = 258 < 16 + 256)
		if (__shfl_sync(full, (int)pend, v)) {
			const int pc = bi == 0 ? c0 : bi == 1 ? c1 : bi == 2 ? c2 : c3;
			const uint32_t ca = (uint32_t)__shfl_sync(full, pc, v) + woff + 16u + 8u * (uint32_t)lane;
			const uint32_t sa = (uint32_t)(s0 + v) + woff + 16u + 8u * (uint32_t)lane;
			int first = 8;
			if (16 + 8 * lane < kMaxMatch) {
				uint32_t a0, a1, b0, b1;
				fast_load8(in, ca, a0, a1);
				fast_load8(in, sa, b0, b1);
				first = fast_lcp8(a0, a1, b0, b1);
			}
			const uint32_t mm = __ballot_sync(full, first < 8);
			const int fl = mm ? __ffs((int)mm) - 1 : 0;
			const int ff = __shfl_sync(full, first, fl);
			int ll = mm ? 16 + 8 * fl + ff : kMaxMatch;
			if (ll > kMaxMatch) ll = kMaxMatch;
			if (lane == v) {
				pend = false;
				if (ll > best) {
					best = ll;
					bestc = pc;
					if (best >= lp.nice) go = false;
				}
				++bi;
				if (go && bi == nb && cand == 0) go = false;
			}
		}
		// replay: the cursor passes every lane whose walk is complete
		const uint32_t fin = __ballot_sync(full, !go);
		if ((fin >> v) & 1u) {
			const uint32_t litm = __ballot_sync(full, active && best < kMinMatch);
			const uint32_t shortm = __ballot_sync(full, best >= kMinMatch && best <= lp.lazy);
			const uint32_t e0 = __ballot_sync(full, best & 1), e1 = __ballot_sync(full, best & 2), e2 = __ballot_sync(full, best & 4);
			uint32_t bad = N ? __ballot_sync(full, (used & N) != 0) : 0u;
			while (v < nl && ((fin >> v) & 1u)) {
				if ((bad >> v) & 1u) {
					stop = true;
					break;
				}
				if ((litm >> v) & 1u) {
					const uint32_t r = ~((litm & fin & ~bad) >> v); // a run of literals
					const int run = r ? __ffs((int)r) - 1 : 32 - v;
					visited |= (run >= 32 ? full : ((1u << run) - 1u)) << v;
					v += run;
					last_long = 0;
				} else if ((shortm >> v) & 1u) {
					const int L = (int)(((e0 >> v) & 1u) | (((e1 >> v) & 1u) << 1) | (((e2 >> v) & 1u) << 2));
					if (v + L > nl) { // its inner positions would need inserting behind the group: the next step takes it
						stop = true;
						break;
					}
					visited |= 1u << v;
					v += L;
					last_long = 0;
				} else {
					const int L = __shfl_sync(full, best, v);
					visited |= 1u << v;
					const int lo_b = v + 1, hi_b = v + L < 32 ? v + L : 32; // positions v+1 .. v+L-1 are not inserted
					if (hi_b > lo_b) N |= (hi_b >= 32 ? full : ((1u << hi_b) - 1u)) & ~((1u << lo_b) - 1u);
					if ((N >> lane) & 1u) { // covered: nobody will ask for this lane's result
						go = false;
						pend = false;
					}
					bad = __ballot_sync(full, (used & N) != 0);
					v += L;
					last_long = 1;
				}
			}
			if (stop || v >= nl) break;
		}
	}
	const int len = best >= kMinMatch ? best : 0;
	// commit
	const uint32_t below = v >= 32 ? full : ((1u << v) - 1u);
	const uint32_t ins = below & ~N & (nl >= 32 ? full : ((1u << nl) - 1u));
	const bool inserted = (ins >> lane) & 1u;
	if (inserted) {
		if (N) {
			const uint32_t pi = same & ins & lt;
			prev[q & 32767] = (uint16_t)(pi ? s0 + (31 - __clz((int)pi)) : hh);
		}
		if (((same & ins) >> lane) == 1u) head[h] = (uint16_t)q;
	}
	if ((visited >> lane) & 1u)
		sout[total + (uint32_t)__popc(visited & lt)] = len ? sym_match((uint32_t)len, (uint32_t)(q - bestc)) : sym_lit(lo & 255u);
	const uint32_t vm = __ballot_sync(full, ((visited >> lane) & 1u) && len != 0);
	if (vm) match_start = __shfl_sync(full, bestc, 31 - __clz((int)vm));
	if (!last_long) last_h = (int)__shfl_sync(full, h, (v - 1) & 31);
	const int nv = __popc(visited);
	total += (uint32_t)nv;
	nsym += (uint32_t)nv;
	s0 += v;
	la -= v;
	__syncwarp();
	return last_long;
}

// B200Z_PARSE_WARM=<positions> (0 .. 4096): how far in front of its first position a parse chunk starts (0: every chunk enters
// with the clean guess and k_parse_fix parses again at most boundaries, as in round 1; for tests and timing)
static int parse_warm() {
	const char *e = getenv("B200Z_PARSE_WARM");
	if (!e) return kParseWarm;
	const long v = atol(e);
	return v < 0 ? 0 : v > 4096 ? 4096 : (int)v;
}

// B200Z_FAST_GROUP=0 keeps every loop top on lane 0 (the serial statement; for measurements and for the tests that compare)
static int fast_group_enabled() {
	const char *e = getenv("B200Z_FAST_GROUP");
	return !(e && e[0] == '0');
}

// One stream's DeflateFast run by one warp.  head[] (32768 entries, read once per loop top) lives in the CTA's slot of a
// global pool and stays in L2; prev[] (read for every chain member) is the CTA's shared memory.
__device__ __forceinline__ void fast_stream(const int stream, const int lane, uint16_t *head, uint16_t *prev, const uint8_t *__restrict__ in,
                                            uint32_t *__restrict__ sym, const int64_t *__restrict__ in_off,
                                            const int64_t *__restrict__ in_len, uint32_t *__restrict__ nsyms,
                                            uint32_t *__restrict__ nblocks, const uint32_t *__restrict__ blk_off,
                                            uint32_t *__restrict__ blk_start, uint32_t *__restrict__ blk_ptop,
                                            const uint32_t *__restrict__ hist, const LevelParams &lp, int strategy, int end_mode,
                                            int prev_entries, const uint32_t *__restrict__ sched, const uint32_t *__restrict__ sched_off,
                                            const int32_t *__restrict__ undrained, uint8_t *const *__restrict__ fstate, int cont,
                                            int group, uint2 *__restrict__ fcut) {
	// prev[] is indexed by window position & 32767; when no stream of the batch is longer than prev_entries - 2 bytes the
	// positions never reach prev_entries, so the table (and the CTA's shared-memory footprint) can be that much smaller
	// and more CTAs share an SM.  (Plans that carry engine state between segments use whole tables.)
	const uint32_t n = (uint32_t)in_len[stream];
	const int64_t off = in_off[stream];
	uint32_t *sout = sym + off;
	uint32_t *bstart = blk_start + blk_off[stream];
	uint32_t *bptop = blk_ptop + blk_off[stream];
	uint8_t *st = fstate[stream]; // engine state carried between the segments of this stream (b200z_history.engine_state)
	const bool resume = cont != 0 && st != nullptr;
	FastEngine e;
	if (resume) {
		// the stream goes on behind a Flush(): tables and scalars as the previous segment's run left them
		const uint4 *src = reinterpret_cast<const uint4 *>(st);
		for (int i = lane; i < 65536 / 16; i += 32) reinterpret_cast<uint4 *>(head)[i] = src[i];
		for (int i = lane; i < 65536 / 16; i += 32) reinterpret_cast<uint4 *>(prev)[i] = src[65536 / 16 + i];
		__syncwarp();
		FastCarry c = *reinterpret_cast<const FastCarry *>(st + 131072);
		fe_load(e, c, in + off, n, hist[stream], head, prev);
	} else {
		for (int i = lane; i < 65536 / 16; i += 32) reinterpret_cast<uint4 *>(head)[i] = make_uint4(0u, 0u, 0u, 0u);
		for (int i = lane; i < prev_entries / 2; i += 32) reinterpret_cast<uint32_t *>(prev)[i] = 0;
		__syncwarp();
		fe_init(e, in + off, n, head, prev);
		if (lane == 0) fe_set_dictionary(e, hist[stream]); // preset dictionary in front of the data (0 = none)
	}
	e.coop = group ? 2 : 1;
	// the SetInput schedule of the segment (fe_run in b200z_core.cuh is the serial statement of this loop, the open run's
	// included)
	const uint32_t *cum = sched + sched_off[stream];
	const int nsched = (int)(sched_off[stream + 1] - sched_off[stream]);
	const int nc = nsched > 0 ? nsched : 1;
	const bool open = end_mode == B200Z_END_NONE;
	const bool busy_last = undrained[stream] == 0 || open;
	uint32_t seg_base = 0, seg_end = 0;
	if (lane == 0) {
		seg_base = fe_stream_pos(e.slides, e.blockStart);
		seg_end = 32768u * e.slides - 1u - e.woff + e.slot_len;
		e.n = nsched > 0 ? seg_base + cum[0] : seg_end;
	}
	// an open run: the engine right behind the last block that closed is the next run's entry.  Tables and scalars are
	// copied at every close that lies within one block's reach of the end of the input (the last one always does: behind it
	// fewer than 16384 symbols of at most 258 bytes each follow, then less than MIN_LOOKAHEAD is left)
	bool closed = false;
	uint32_t cut_cov = 0, cut_call = 0;
	if (open && lane == 0) fcut[stream] = make_uint2(0u, 0u);
	uint32_t total = 0, nblk = 0;
#ifdef B200Z_FAST_STATS
	uint32_t st_steps = 0, st_pos = 0, st_lanes = 0;
#endif
	int ci = 0;
	int phase = (nc == 1 && !busy_last) ? 1 : 0; // 0: BUSY_STATE drain of chunk ci, 1: Flush()/Finish()
	bool in_deflate = false; // re-entering DeflateFast after a cooperative slide must not run FillWindow again
	const bool finish = end_mode == B200Z_END_FINISH;
	for (;;) {
		int r = kFeTrue;
		if (lane == 0) {
			bool filled = true;
			if (!in_deflate) filled = fe_fill_window(e);
			if (!filled) {
				r = kFeNeedSlide;
			} else {
				in_deflate = true;
				// engine.Deflate(flush, finish): canFlush = flush && inputOff == inputEnd (DeflaterEngine.cs:104-137)
				r = fe_deflate_fast(
				    e, phase == 1 && e.inputOff == e.n, phase == 1 && finish, lp, strategy, [&](uint32_t s2) { sout[total++] = s2; },
				    [&](uint32_t start, bool ok, bool) {
					    bstart[nblk] = start;
					    bptop[nblk] = ok ? 0xFFFFFFFEu : 0xFFFFFFFFu; // storedOffset sign decided by the engine (trap T4)
					    ++nblk;
					    closed = true;
				    });
				if (r != kFeNeedSlide && r != kFeGroup) in_deflate = false;
			}
		}
		r = __shfl_sync(0xffffffffu, r, 0);
		if (r == kFeGroup) {
			// steady-state loop tops ahead: the warp takes them in groups (fast_group_step) until a slide, a full block or the
			// end of the lookahead comes near; lane 0's engine is brought in step afterwards
			int s0 = __shfl_sync(0xffffffffu, e.strstart, 0), la = __shfl_sync(0xffffffffu, e.lookahead, 0);
			uint32_t nsym = __shfl_sync(0xffffffffu, e.nsym, 0);
			const uint32_t woff = __shfl_sync(0xffffffffu, e.woff, 0);
			total = __shfl_sync(0xffffffffu, total, 0);
			int last_h = 0, match_start = __shfl_sync(0xffffffffu, e.matchStart, 0), last_long = 0, nl;
			while ((nl = fe_group_lanes(s0, la, nsym)) >= kFeGroupMin) {
#ifdef B200Z_FAST_STATS
				const int s_before = s0;
#endif
				last_long = fast_group_step(in + off, woff, head, prev, lp, lane, nl, s0, la, nsym, sout, total, last_h, match_start);
#ifdef B200Z_FAST_STATS
				++st_steps;
				st_pos += (uint32_t)(s0 - s_before);
				st_lanes += (uint32_t)(s0 - s_before < 32 ? s0 - s_before : 32);
#endif
			}
			if (lane == 0) {
				e.strstart = s0;
				e.lookahead = la;
				e.nsym = nsym;
				e.matchStart = match_start;
				e.matchLen = kMinMatch - 1;
				if (last_long)
					fe_update_hash(e); // :712-714 (lookahead >= MIN_MATCH - 1 holds: it was >= 262 before a match of <= 258)
				else
					e.ins_h = last_h;
				// back at the top of DeflateFast's loop: `while (lookahead >= MIN_LOOKAHEAD || flush)` (:658)
				const bool flush = phase == 1 && e.inputOff == e.n;
				if (e.lookahead < kMaxMatch + kMinMatch + 1 && !flush) {
					in_deflate = false; // the loop ends, DeflateFast returns true (:738)
					r = kFeTrue;
				}
			}
			r = __shfl_sync(0xffffffffu, r, 0);
			if (r == kFeGroup) continue; // lane 0 goes on inside DeflateFast (in_deflate is still set)
		}
		r = __shfl_sync(0xffffffffu, r, 0);
		if (open) {
			// (a block closes only on lane 0's serial path: group steps stop one symbol short of a full block)
			int snap = 0;
			if (lane == 0 && closed) {
				closed = false;
				cut_cov = (uint32_t)e.blockStart + e.woff - hist[stream];
				cut_call = (uint32_t)ci;
				snap = e.slot_len - ((uint32_t)e.blockStart + e.woff) <= (uint32_t)(kBlockSyms * kMaxMatch + kMaxMatch + kMinMatch + 1);
				if (snap) {
					FastCarry c;
					fe_save(e, c);
					*reinterpret_cast<FastCarry *>(st + 131072) = c;
				}
			}
			if (__shfl_sync(0xffffffffu, snap, 0)) {
				__syncwarp();
				uint4 *dst = reinterpret_cast<uint4 *>(st);
				for (int i = lane; i < 65536 / 16; i += 32) dst[i] = reinterpret_cast<const uint4 *>(head)[i];
				for (int i = lane; i < 65536 / 16; i += 32) dst[65536 / 16 + i] = reinterpret_cast<const uint4 *>(prev)[i];
				__syncwarp();
			}
		}
		if (r == kFeNeedSlide) {
			// SlideWindow (DeflaterEngine.cs:441-462): scalars by lane 0, both tables by the warp
			if (lane == 0) fe_slide_scalars(e);
			for (int t = 0; t < 2; t++) { // 2 entries per 32-bit word (a slide means a stream beyond 64 KiB: whole tables)
				uint32_t *tab = reinterpret_cast<uint32_t *>(t ? prev : head);
				for (int i = lane; i < 16384; i += 32) {
					const uint32_t v = tab[i];
					uint32_t lo = v & 0xFFFFu, hi = v >> 16;
					lo = lo >= 32768u ? lo - 32768u : 0u;
					hi = hi >= 32768u ? hi - 32768u : 0u;
					tab[i] = lo | (hi << 16);
				}
			}
			__syncwarp();
			continue;
		}
		if (r == kFeFalse) {
			if (phase == 1) break;
			// chunk ci is drained ("needs input"): the next SetInput, or Flush()/Finish() (an open run ends here)
			++ci;
			if (ci < nc) {
				if (lane == 0) e.n = seg_base + cum[ci];
				if (ci == nc - 1 && !busy_last) phase = 1;
			} else {
				if (open) break;
				phase = 1;
			}
		}
	}
	if (lane == 0) {
		if (open) {
			// the blocks in front of the cut are written; the last one ends where the next run's data starts
			total = nblk * (uint32_t)kBlockSyms;
			bstart[nblk] = cut_cov + hist[stream];
			if (nblk) fcut[stream] = make_uint2(cut_cov, cut_call);
		}
		nsyms[stream] = total;
		nblocks[stream] = nblk;
#ifdef B200Z_FAST_STATS
		printf("k_fast stream %d: n %u, group steps %u, positions by groups %u (%.1f per step, %.1f lanes used), symbols %u\n", stream, n,
		       st_steps, st_pos, st_steps ? (double)st_pos / st_steps : 0.0, st_steps ? (double)st_lanes / st_steps : 0.0, total);
#endif
	}
	if (st && !open) {
		// what the next segment of this stream starts from
		__syncwarp();
		uint4 *dst = reinterpret_cast<uint4 *>(st);
		for (int i = lane; i < 65536 / 16; i += 32) dst[i] = reinterpret_cast<const uint4 *>(head)[i];
		const int words = prev_entries * 2 / 16;
		for (int i = lane; i < words; i += 32) dst[65536 / 16 + i] = reinterpret_cast<const uint4 *>(prev)[i];
		for (int i = words + lane; i < 65536 / 16; i += 32) dst[65536 / 16 + i] = make_uint4(0u, 0u, 0u, 0u);
		if (lane == 0) {
			FastCarry c;
			fe_save(e, c);
			*reinterpret_cast<FastCarry *>(st + 131072) = c;
		}
	}
}

// persistent CTAs of one warp: streams are taken off a counter, so a batch of uneven streams keeps every CTA busy
__global__ void __launch_bounds__(32)
    k_fast(const uint8_t *__restrict__ in, uint32_t *__restrict__ sym, const int64_t *__restrict__ in_off,
           const int64_t *__restrict__ in_len, uint32_t *__restrict__ nsyms, uint32_t *__restrict__ nblocks,
           const uint32_t *__restrict__ blk_off, uint32_t *__restrict__ blk_start, uint32_t *__restrict__ blk_ptop,
           const uint32_t *__restrict__ hist, LevelParams lp, int strategy, int end_mode, int prev_entries,
           const uint32_t *__restrict__ sched, const uint32_t *__restrict__ sched_off, const int32_t *__restrict__ undrained,
           uint8_t *const *__restrict__ fstate, int cont, int group, int nstreams, uint16_t *__restrict__ head_pool,
           uint32_t *__restrict__ counter, uint2 *__restrict__ fcut) {
	extern __shared__ __align__(16) uint8_t fsm[];
	uint16_t *prev = reinterpret_cast<uint16_t *>(fsm);
	// head_pool == nullptr: a batch of at most one stream per SM -- head[] sits behind prev[] in shared memory (one CTA per
	// SM then, whose L1 holds the stream's window: 1.7x faster per stream than with three CTAs sharing the SM)
	uint16_t *head = head_pool ? head_pool + 32768ll * blockIdx.x : prev + prev_entries;
	const int lane = threadIdx.x;
	for (;;) {
		int stream = 0;
		if (lane == 0) stream = (int)atomicAdd(counter, 1u);
		stream = __shfl_sync(0xffffffffu, stream, 0);
		if (stream >= nstreams) break;
		fast_stream(stream, lane, head, prev, in, sym, in_off, in_len, nsyms, nblocks, blk_off, blk_start, blk_ptop, hist, lp, strategy,
		            end_mode, prev_entries, sched, sched_off, undrained, fstate, cont, group, fcut);
		__syncwarp();
	}
}

// ------------------------------------------------------------------------------------------------
// Level 0: DeflateStored.  Block boundaries are pure bookkeeping (stored_run, computed when the plan is built);
// the kernel writes 1 header byte, LEN, ~LEN and copies the bytes (FlushStoredBlock, DeflaterHuffman.cs:766-779).
// ------------------------------------------------------------------------------------------------
struct StoredBlock {
	int32_t stream;
	uint32_t src;     // first input byte inside the stream
	uint32_t len;
	uint32_t last;
	uint64_t dst;     // byte offset of the block inside the stream's output slot
};

__global__ void __launch_bounds__(256)
    k_stored(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, const int64_t *__restrict__ in_off,
             const int64_t *__restrict__ out_off, const StoredBlock *__restrict__ blocks) {
	const StoredBlock b = blocks[blockIdx.x];
	const uint8_t *src = in + in_off[b.stream] + b.src;
	uint8_t *dst = out + out_off[b.stream] + b.dst;
	if (threadIdx.x == 0) {
		dst[0] = (uint8_t)(b.last ? 1 : 0); // 3 header bits (STORED_BLOCK << 1 | last) then AlignToByte
		dst[1] = (uint8_t)b.len;
		dst[2] = (uint8_t)(b.len >> 8);
		dst[3] = (uint8_t)~b.len;
		dst[4] = (uint8_t)(~b.len >> 8);
	}
	for (uint32_t i = threadIdx.x; i < b.len; i += blockDim.x) dst[5 + i] = src[i];
}

__global__ void k_set_results(int n, const int64_t *__restrict__ lens, int64_t *__restrict__ out_len, int32_t *__restrict__ status,
                              int64_t *__restrict__ out_bits) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	out_len[i] = lens[i];
	status[i] = B200Z_OK;
	if (out_bits) out_bits[i] = 8 * lens[i];
}

// ------------------------------------------------------------------------------------------------
// K4: per-block histograms, the reference's Huffman construction and the block type decision.
// One CTA of two warps per block.  Only the heap of each Tree.BuildTree and BuildLength (whose tie-breaks decide the
// bytes) run on one lane, the literal and the distance tree on one lane of each warp; everything around them is
// order-free and runs warp-wide: the histogram, CalcBLFreq and the header's code-length string (per run of equal code
// lengths, walk_code_run), the cost sums and BuildCodes.  What plan_block_finish() does serially for the CPU model.
// The footprint (8.3 KiB of shared memory, <= 40 registers, no stack frame) keeps 24 CTAs on an SM: the 7,213 blocks of
// bench.py's 1024 x 256 KiB at level 6 run in 2.3 waves of 3,168 CTAs on an H100.
// ------------------------------------------------------------------------------------------------
constexpr int kPlanThreads = 64;

__device__ __forceinline__ uint32_t lanes_below() {
	return (1u << (threadIdx.x & 31)) - 1u;
}
__device__ __forceinline__ void or_hdr(uint32_t *w, uint32_t pos, uint32_t v, int count) {
	const uint32_t idx = pos >> 5, sh = pos & 31;
	atomicOr(w + idx, v << sh);
	if (sh + (uint32_t)count > 32) atomicOr(w + idx + 1, v >> (32 - sh));
}
// Tree.BuildCodes warp-wide: symbol i gets nextCode[len] + (the symbols in front of it with the same length) << (16 - len).
// next[0..maxLength) is the per-length start from the bl_counts, advanced chunk by chunk.
__device__ void build_codes_warp(const uint8_t *length, const int *bl_counts, int maxLength, int numCodes, uint16_t *codes,
                                 int *next) {
	const int lane = threadIdx.x & 31;
	if (lane == 0) {
		int code = 0;
		for (int bits = 0; bits < maxLength; bits++) {
			next[bits] = code;
			code += bl_counts[bits] << (15 - bits);
		}
	}
	__syncwarp();
	for (int base = 0; base < numCodes; base += 32) {
		const int i = base + lane;
		const int bits = i < numCodes ? length[i] : 0;
		const uint32_t peers = __match_any_sync(0xffffffffu, bits);
		if (i < numCodes)
			codes[i] = bits ? (uint16_t)bit_reverse16((uint32_t)(next[bits - 1] + (__popc(peers & lanes_below()) << (16 - bits)))) : 0;
		__syncwarp();
		if (bits && (peers >> lane) == 1u) next[bits - 1] += __popc(peers) << (16 - bits); // the group's last lane
		__syncwarp();
	}
}
// sum over a warp
__device__ __forceinline__ int warp_sum(int v) {
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	return v;
}

__global__ void __launch_bounds__(kPlanThreads, 24)
    k_plan(const uint32_t *__restrict__ sym, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
           const uint32_t *__restrict__ nsyms, const uint32_t *__restrict__ nblocks, const uint32_t *__restrict__ blk_off,
           const int32_t *__restrict__ blk_desc, const uint32_t *__restrict__ blk_start, const uint32_t *__restrict__ blk_ptop,
           BlockMeta *__restrict__ meta, BlockTables *__restrict__ tables, const int64_t *__restrict__ bias, int end_mode) {
	__shared__ int s_lit[kLiteralNum];
	__shared__ int s_dist[kDistNum];
	__align__(8) __shared__ int s_scratch[tree_scratch_ints(kLiteralNum)]; // the literal tree, then the header and the runs
	__align__(8) __shared__ int s_scratch2[tree_scratch_ints(kDistNum)];   // the distance tree, then the bit-length tree
	__shared__ int s_blc[3][16];  // bl_counts of the literal, distance and bit-length trees
	__shared__ int s_next[3][16]; // BuildCodes' nextCode, per tree
	__shared__ int s_bl_freqs[kBitlenNum];
	__shared__ uint8_t s_bl_len[kBitlenNum + 1];
	__shared__ uint16_t s_bl_codes[kBitlenNum + 1];
	__shared__ int s_v[6]; // extra bits, literal numCodes, distance numCodes, static_len, dynamic body bits, runs
	// the members of BlockTables in front of hdr (the header words live in s_scratch, where the literal tree was built);
	// s_tab.hdr is never touched
	__align__(16) __shared__ uint8_t s_tabmem[offsetof(BlockTables, hdr)];
	BlockTables &s_tab = *reinterpret_cast<BlockTables *>(s_tabmem);
	uint32_t *hdr = reinterpret_cast<uint32_t *>(s_scratch);
	const int g = blockIdx.x;
	const int stream = blk_desc[g];
	const uint32_t b = (uint32_t)g - blk_off[stream];
	const uint32_t nb = nblocks[stream];
	if (b >= nb) return;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const uint32_t ns = nsyms[stream];
	const uint32_t s0 = b * (uint32_t)kBlockSyms;
	const uint32_t s1 = (ns - s0 > (uint32_t)kBlockSyms) ? s0 + kBlockSyms : ns;
	const uint32_t *sp = sym + in_off[stream];
	for (int i = tid; i < kLiteralNum; i += kPlanThreads) s_lit[i] = 0;
	for (int i = tid; i < kDistNum; i += kPlanThreads) s_dist[i] = 0;
	if (tid < kBitlenNum) s_bl_freqs[tid] = 0;
	if (tid == 0) s_v[0] = 0;
	__syncthreads();
	int extra = 0;
	for (uint32_t i0 = s0 + tid; i0 < s1; i0 += 8 * kPlanThreads) {
		// eight independent loads in flight per thread (ncu: the one-load-per-trip loop sat on long_scoreboard)
		uint32_t sv[8];
#pragma unroll
		for (int k = 0; k < 8; k++) {
			const uint32_t i = i0 + (uint32_t)k * kPlanThreads;
			sv[k] = i < s1 ? __ldg(sp + i) : 0xFFFFFFFFu;
		}
#pragma unroll
		for (int k = 0; k < 8; k++) {
			const uint32_t s = sv[k];
			if (s == 0xFFFFFFFFu) continue; // (not a symbol: distances stop at 32506)
			if (sym_dist(s) == 0) {
				atomicAdd(&s_lit[s & 0xFF], 1);
			} else {
				const int lc = lcode((int)(s & 0xFF)), dc = dcode((int)sym_dist(s) - 1);
				atomicAdd(&s_lit[lc], 1);
				atomicAdd(&s_dist[dc], 1);
				extra += tally_extra_bits(lc, dc);
			}
		}
	}
	extra = warp_sum(extra);
	if (lane == 0 && extra) atomicAdd(&s_v[0], extra);
	__syncthreads();
	if (tid == 0) s_lit[256] += 1; // FlushBlock: literalTree.freqs[EOF_SYMBOL]++ (:790)
	__syncthreads();
	// the two big trees are independent: build them on two warps at once
	if (tid == 0) s_v[1] = build_tree(s_lit, kLiteralNum, 257, 15, s_tab.lit_len, s_blc[0], s_scratch);
	if (tid == 32) s_v[2] = build_tree(s_dist, kDistNum, 1, 15, s_tab.dist_len, s_blc[1], s_scratch2);
	__syncthreads();
	const int lit_nc = s_v[1], dist_nc = s_v[2], nlen = lit_nc + dist_nc;
	uint16_t *runs = reinterpret_cast<uint16_t *>(hdr + kHdrWords); // first code length of every run, then nlen
	auto len_at = [&](int j) -> int { return j < lit_nc ? s_tab.lit_len[j] : s_tab.dist_len[j - lit_nc]; };
	if (warp == 0) {
		// CalcBLFreq: the runs of equal code lengths (the walk restarts at the distance lengths), then their symbols
		int nruns = 0;
		for (int base = 0; base < nlen; base += 32) {
			const int j = base + lane;
			const bool start = j < nlen && (j == 0 || j == lit_nc || len_at(j) != len_at(j - 1));
			const uint32_t m = __ballot_sync(0xffffffffu, start);
			if (start) runs[nruns + __popc(m & lanes_below())] = (uint16_t)j;
			nruns += __popc(m);
		}
		if (lane == 0) {
			runs[nruns] = (uint16_t)nlen;
			s_v[5] = nruns;
		}
		__syncwarp();
		for (int k = lane; k < nruns; k += 32)
			walk_code_run(len_at(runs[k]), runs[k + 1] - runs[k], [&](int s) { atomicAdd(&s_bl_freqs[s], 1); }, [](int, int) {});
	} else {
		// the cost sums that do not need the bit-length tree
		int st = 0, dyn = 0;
		for (int i = lane; i < kLiteralNum; i += 32) {
			st += s_lit[i] * static_llen(i);
			dyn += s_lit[i] * s_tab.lit_len[i];
		}
		if (lane < kDistNum) {
			st += s_dist[lane] * 5;
			dyn += s_dist[lane] * s_tab.dist_len[lane];
		}
		st = warp_sum(st);
		dyn = warp_sum(dyn);
		if (lane == 0) {
			s_v[3] = s_v[0] + st;
			s_v[4] = s_v[0] + dyn;
		}
		for (int i = lane; i < kHdrWords; i += 32) hdr[i] = 0;
	}
	__syncthreads();
	if (tid == 0) build_tree(s_bl_freqs, kBitlenNum, 4, 7, s_bl_len, s_blc[2], s_scratch2);
	__syncthreads();
	int blTreeCodes = 4;
	for (int i = 18; i > blTreeCodes; i--) {
		if (s_bl_len[bl_order(i)] > 0) blTreeCodes = i + 1;
	}
	int bl_cost = 0;
	for (int i = 0; i < kBitlenNum; i++) bl_cost += s_bl_freqs[i] * s_bl_len[i];
	const int static_len = s_v[3], body = s_v[4];
	int opt_len = 14 + blTreeCodes * 3 + bl_cost + body;
	if (opt_len >= static_len) opt_len = static_len; // force static trees

	const uint32_t *bstart = blk_start + blk_off[stream];
	const uint32_t byte_start = bstart[b];
	const uint32_t n = (uint32_t)in_len[stream];
	// (an open run's last written block ends at a cut, like every block in front of it)
	const uint32_t byte_len = ((b + 1 < nb || end_mode == B200Z_END_NONE) ? bstart[b + 1] : n) - byte_start;
	// storedOffset is window relative and goes negative once the block start has been slid out (trap T4)
	const uint32_t ptop = blk_ptop[blk_off[stream] + b];
	const long long ab = bias[stream]; // absolute stream offset of buffer position 0
	long long storedOffset = (long long)byte_start + ab + 1 - 32768ll * (long long)slides_done((uint32_t)(ptop + ab));
	if (ptop >= 0xFFFFFFFEu) storedOffset = ptop == 0xFFFFFFFEu ? 0 : -1; // levels 1-4: decided by k_fast
	const int last = (b + 1 == nb) && end_mode == B200Z_END_FINISH;
	const int type = block_type(storedOffset >= 0, (int)byte_len, opt_len, static_len);
	uint32_t hdr_bits = 3, body_bits = 0;
	if (type == 0) {
		if (tid == 0) hdr[0] = (uint32_t)((0 << 1) + last);
	} else if (type == 1) {
		body_bits = (uint32_t)static_len;
		if (tid == 0) hdr[0] = (uint32_t)((1 << 1) + last);
		for (int i = tid; i < kLiteralNum; i += kPlanThreads) {
			s_tab.lit_len[i] = (uint8_t)static_llen(i);
			s_tab.lit_codes[i] = (uint16_t)static_lcode(i);
		}
		if (tid < kDistNum) {
			s_tab.dist_len[tid] = 5;
			s_tab.dist_codes[tid] = (uint16_t)static_dcode(tid);
		}
	} else {
		// SendAllTrees (:676-696)
		body_bits = (uint32_t)body;
		if (warp == 0) {
			build_codes_warp(s_tab.lit_len, s_blc[0], 15, lit_nc, s_tab.lit_codes, s_next[0]);
		} else {
			build_codes_warp(s_tab.dist_len, s_blc[1], 15, dist_nc, s_tab.dist_codes, s_next[1]);
			build_codes_warp(s_bl_len, s_blc[2], 7, kBitlenNum, s_bl_codes, s_next[2]);
		}
		__syncthreads();
		const uint32_t pre = 17 + 3 * (uint32_t)blTreeCodes;
		if (warp == 0) {
			// the code-length string: every run's bits at its prefix-summed offset
			const int nruns = s_v[5];
			uint32_t off = pre;
			for (int base = 0; base < nruns; base += 32) {
				const int k = base + lane;
				int v = 0, r = 0;
				uint32_t nbits = 0;
				if (k < nruns) {
					v = len_at(runs[k]);
					r = runs[k + 1] - runs[k];
					walk_code_run(v, r, [&](int s) { nbits += s_bl_len[s]; }, [&](int, int nb) { nbits += (uint32_t)nb; });
				}
				uint32_t incl = nbits;
				for (int o = 1; o < 32; o <<= 1) {
					const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
					if (lane >= o) incl += t;
				}
				uint32_t pos = off + incl - nbits;
				if (k < nruns)
					walk_code_run(
					    v, r,
					    [&](int s) {
						    or_hdr(hdr, pos, s_bl_codes[s], s_bl_len[s]);
						    pos += s_bl_len[s];
					    },
					    [&](int x, int nb) {
						    or_hdr(hdr, pos, (uint32_t)x, nb);
						    pos += (uint32_t)nb;
					    });
				off += __shfl_sync(0xffffffffu, incl, 31);
			}
			hdr_bits = off;
		} else {
			if (lane == 0)
				or_hdr(hdr, 0,
				       (uint32_t)((2 << 1) + last) | (uint32_t)(lit_nc - 257) << 3 | (uint32_t)(dist_nc - 1) << 8 |
				           (uint32_t)(blTreeCodes - 4) << 13,
				       17);
			if (lane < blTreeCodes) or_hdr(hdr, 17 + 3 * (uint32_t)lane, s_bl_len[bl_order(lane)], 3);
		}
	}
	if (tid == 0) {
		BlockMeta m;
		m.byte_start = byte_start;
		m.byte_len = byte_len;
		m.nsyms = s1 - s0;
		m.hdr_bits = hdr_bits;
		m.body_bits = body_bits;
		m.type = (uint32_t)type;
		m.bit_off = 0;
		meta[g] = m;
	}
	__syncthreads();
	// copy the tables out
	constexpr int kHdrOff = (int)offsetof(BlockTables, hdr) / 4;
	static_assert(offsetof(BlockTables, hdr) % 4 == 0, "");
	const uint32_t *src = reinterpret_cast<const uint32_t *>(s_tabmem);
	uint32_t *dst = reinterpret_cast<uint32_t *>(&tables[g]);
	for (int i = tid; i < kHdrOff + kHdrWords; i += kPlanThreads) dst[i] = i < kHdrOff ? src[i] : hdr[i - kHdrOff];
}

__device__ __forceinline__ void or_bits(uint32_t *out_words, uint64_t bitpos, uint64_t bits, int nbits) {
	// nbits <= 57; spreads over at most three 32-bit words
	if (nbits == 0) return;
	const uint64_t idx = bitpos >> 5;
	const uint32_t sh = (uint32_t)(bitpos & 31);
	const uint64_t lo = bits << sh;
	atomicOr(out_words + idx, (uint32_t)lo);
	if (sh + nbits > 32) {
		atomicOr(out_words + idx + 1, (uint32_t)(lo >> 32));
		if (sh + nbits > 64) atomicOr(out_words + idx + 2, (uint32_t)(bits >> (64 - sh)));
	}
}

// ------------------------------------------------------------------------------------------------
// K5: bit offset of every block inside its stream (stored blocks byte-align), end-of-stream bits, sizes.
// ------------------------------------------------------------------------------------------------
__global__ void k_scan(int nstreams, const uint32_t *__restrict__ nblocks, const uint32_t *__restrict__ blk_off,
                       BlockMeta *__restrict__ meta, uint8_t *__restrict__ out, const int64_t *__restrict__ out_off,
                       const int64_t *__restrict__ out_cap, int64_t *__restrict__ out_len, int32_t *__restrict__ status,
                       int64_t *__restrict__ out_bits, const uint32_t *__restrict__ bit_base, int end_mode) {
	const int stream = blockIdx.x * blockDim.x + threadIdx.x;
	if (stream >= nstreams) return;
	const uint32_t nb = nblocks[stream];
	BlockMeta *m = meta + blk_off[stream];
	uint64_t cur = bit_base[stream]; // 0..7: a continued stream starts inside the byte the previous segment ended in
	for (uint32_t b = 0; b < nb; b++) {
		m[b].bit_off = cur;
		if (m[b].type == 0) cur = ((cur + 3 + 7) & ~7ull) + 32 + 8ull * m[b].byte_len;
		else cur += (uint64_t)m[b].hdr_bits + m[b].body_bits;
	}
	uint64_t tail0 = cur;
	int ntail10 = 0; // number of 10-bit empty static blocks: "WriteBits(2, 10)" (Deflater.cs:486-504)
	if (end_mode == B200Z_END_FLUSH || end_mode == B200Z_END_FLUSH_FINISH) {
		int neededbits = 8 + (int)((0 - cur) & 7);
		while (neededbits > 0) {
			++ntail10;
			cur += 10;
			neededbits -= 10;
		}
	}
	if (end_mode == B200Z_END_FLUSH_FINISH) cur += 10; // the final empty static block (3, 10 bits)
	const uint64_t nbytes = (cur + 7) >> 3; // FINISHING_STATE: pending.AlignToByte() (Deflater.cs:507)
	if ((int64_t)(((nbytes + 3) >> 2) << 2) > out_cap[stream]) {
		status[stream] = B200Z_E_NOMEM;
		out_len[stream] = 0;
		if (out_bits) out_bits[stream] = 0;
		for (uint32_t b = 0; b < nb; b++) m[b].type = 0xFFu; // tells k_emit to skip
		return;
	}
	uint32_t *ow = reinterpret_cast<uint32_t *>(out + out_off[stream]);
	uint64_t t = tail0;
	for (int i = 0; i < ntail10; i++, t += 10) or_bits(ow, t, 2, 10);
	if (end_mode == B200Z_END_FLUSH_FINISH) or_bits(ow, t, 3, 10);
	status[stream] = B200Z_OK;
	out_len[stream] = (int64_t)nbytes;
	if (out_bits) out_bits[stream] = (int64_t)cur; // exact length; a flushed stream may end inside its last byte
}

// ------------------------------------------------------------------------------------------------
// K6: bit emission.  One CTA per block; symbols are encoded 256 at a time, a block-wide exclusive scan of the code
// lengths gives every symbol its bit position, and the code words are OR-ed into the (zeroed) output words.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_emit(const uint8_t *__restrict__ in, const uint32_t *__restrict__ sym, uint8_t *__restrict__ out,
           const int64_t *__restrict__ in_off, const int64_t *__restrict__ out_off, const uint32_t *__restrict__ nblocks,
           const uint32_t *__restrict__ blk_off, const int32_t *__restrict__ blk_desc, const BlockMeta *__restrict__ meta,
           const BlockTables *__restrict__ tables) {
	__shared__ BlockTables s_tab;
	__shared__ uint32_t s_warp[8];
	__shared__ uint64_t s_base;
	const int g = blockIdx.x;
	const int stream = blk_desc[g];
	const uint32_t b = (uint32_t)g - blk_off[stream];
	if (b >= nblocks[stream]) return;
	const BlockMeta m = meta[g];
	if (m.type == 0xFFu) return;
	uint32_t *ow = reinterpret_cast<uint32_t *>(out + out_off[stream]);
	if (m.type == 0) {
		// FlushStoredBlock (:766-779): 3 header bits, pad to byte, LEN, ~LEN, raw bytes
		const uint8_t *src = in + in_off[stream] + m.byte_start;
		const uint64_t hb = ((m.bit_off + 3 + 7) & ~7ull);
		if (threadIdx.x == 0) {
			or_bits(ow, m.bit_off, tables[g].hdr[0] & 7u, 3);
			or_bits(ow, hb, m.byte_len & 0xFFFFu, 16);
			or_bits(ow, hb + 16, (~m.byte_len) & 0xFFFFu, 16);
		}
		const uint64_t d0 = (hb + 32) >> 3; // byte offset of the payload in the stream's output
		uint8_t *ob = out + out_off[stream];
		// head bytes up to a word boundary and tail bytes go through atomicOr; whole words are plain stores
		const uint32_t len = m.byte_len;
		uint32_t headn = (uint32_t)((4 - (d0 & 3)) & 3);
		if (headn > len) headn = len;
		const uint32_t nwords = (len - headn) >> 2;
		const uint32_t tailn = len - headn - (nwords << 2);
		for (uint32_t i = threadIdx.x; i < headn; i += blockDim.x) or_bits(ow, (d0 + i) << 3, src[i], 8);
		uint32_t *wdst = reinterpret_cast<uint32_t *>(ob + d0 + headn);
		for (uint32_t i = threadIdx.x; i < nwords; i += blockDim.x) {
			const uint8_t *s4 = src + headn + (i << 2);
			wdst[i] = (uint32_t)s4[0] | ((uint32_t)s4[1] << 8) | ((uint32_t)s4[2] << 16) | ((uint32_t)s4[3] << 24);
		}
		for (uint32_t i = threadIdx.x; i < tailn; i += blockDim.x)
			or_bits(ow, (d0 + headn + (nwords << 2) + i) << 3, src[headn + (nwords << 2) + i], 8);
		return;
	}
	{
		const uint4 *src = reinterpret_cast<const uint4 *>(&tables[g]);
		uint4 *dst = reinterpret_cast<uint4 *>(&s_tab);
		for (int i = threadIdx.x; i < (int)(sizeof(BlockTables) / 16); i += blockDim.x) dst[i] = src[i];
	}
	if (threadIdx.x == 0) s_base = m.bit_off + m.hdr_bits;
	__syncthreads();
	// header words
	for (uint32_t i = threadIdx.x; i * 32 < m.hdr_bits; i += blockDim.x) {
		const uint32_t rem = m.hdr_bits - i * 32;
		const int nbw = rem < 32 ? (int)rem : 32;
		uint32_t v = s_tab.hdr[i];
		if (nbw < 32) v &= (1u << nbw) - 1u;
		or_bits(ow, m.bit_off + i * 32ull, v, nbw);
	}
	const uint32_t *sp = sym + in_off[stream] + b * (uint32_t)kBlockSyms;
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	for (uint32_t i0 = 0; i0 < m.nsyms; i0 += blockDim.x) {
		const uint32_t i = i0 + threadIdx.x;
		uint64_t bits = 0;
		int nb = 0;
		if (i < m.nsyms) encode_symbol(sp[i], s_tab.lit_codes, s_tab.lit_len, s_tab.dist_codes, s_tab.dist_len, bits, nb);
		// block-wide exclusive scan of nb
		uint32_t incl = (uint32_t)nb;
		for (int o = 1; o < 32; o <<= 1) {
			uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= o) incl += t;
		}
		if (lane == 31) s_warp[wid] = incl;
		__syncthreads();
		uint32_t woff = 0, tot = 0;
		for (int k = 0; k < 8; k++) {
			const uint32_t v = s_warp[k];
			if (k < wid) woff += v;
			tot += v;
		}
		const uint64_t base = s_base;
		or_bits(ow, base + woff + incl - (uint32_t)nb, bits, nb);
		__syncthreads();
		if (threadIdx.x == 0) s_base = base + tot;
		__syncthreads();
	}
	if (threadIdx.x == 0) or_bits(ow, s_base, s_tab.lit_codes[256], s_tab.lit_len[256]); // EOF_SYMBOL (:750)
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// A plan runs one of three engines, chosen by its level: the lazy parse (5-9), DeflateFast (1-4, k_fast) or DeflateStored
// (0, k_stored).  Each engine has its own part of the plan, laid out by its *_layout function and launched by its *_launch
// function; deflate_plan_build and deflate_plan_run do what is common and pick the engine.
struct DeflatePlan final : b200z_plan {
	// common, per stream (b200z_deflate_plan_create_ex): the history in front of the data, the bits in front of the output
	int hist_kind = 0; // B200Z_HIST_*
	bool check_seeded = false;
	std::vector<int64_t> bias;     // stream position of the slot's first byte (pos_base - history)
	std::vector<uint32_t> bit_base;
	// levels 0-4: the SetInput schedule (cumulative sizes of stream i's calls at sched[sched_off[i] .. sched_off[i + 1]]),
	// and "Flush()/Finish() behind an undrained SetInput"
	std::vector<uint32_t> sched, sched_off;
	std::vector<int32_t> undrained;
	bool cut_ready = false; // an open run has been launched since the plan was made
	int n_ck_tiles = 0;
	Slot<uint32_t> o_hist, o_bitbase;
	Slot<int64_t> o_bias, o_ck_off, o_ck_len;
	Slot<CkTile> o_ck_desc;
	Slot<unsigned long long> o_ck_acc;
	// levels 1-9: the symbols and the blocks they are cut into (blocks_layout)
	int n_blkmax = 0;
	Slot<uint32_t> o_sym, o_blk_off, o_nsyms, o_nblocks, o_blk_start, o_blk_ptop;
	Slot<int32_t> o_blk_desc;
	Slot<BlockMeta> o_meta;
	Slot<BlockTables> o_tables;
	struct { // levels 5-9 (lazy_layout)
		int link_run = 65536; // positions per k_links CTA (B200Z_LINK_RUN)
		uint32_t parse_chunk = 32768;
		int n_runs = 0, n_tiles = 0, n_chunks = 0, n_rgroups = 0;
		std::vector<std::vector<uint8_t>> hist_mask; // (b200z_history.hist_mask; empty: the default)
		Slot<int2> o_run_desc, o_tile_desc, o_rgroups;
		Slot<int64_t> o_hm_off;
		Slot<uint8_t> o_hmask;
		Slot<uint16_t> o_link;
		Slot<uint2> o_mt;
		Slot<uint32_t> o_sym_local, o_rnd_off, o_rnd_symoff;
		Slot<ChunkDesc> o_chunks;
		Slot<RoundRec> o_recs, o_ents;
		Slot<RoundRec> o_entry, o_cut; // per stream: the parse state a run starts from, and where an open run stopped
		std::vector<RoundRec> entry;   // what o_entry holds (b200z_deflate_plan_set_entry; a clean start by default)
	} lazy;
	struct { // levels 1-4 (fast_layout)
		std::vector<uint8_t *> engine_state; // per stream, the engine state carried between its segments (device pointers)
		int prev_entries = 32768;         // k_fast's prev[] size for this batch
		int ctas = 1;                     // k_fast's persistent CTAs (each owns a head[] slot of the pool)
		bool head_smem = false;           // ... or keeps head[] in shared memory (few streams)
		Slot<uint32_t> o_sched, o_sched_off, o_counter;
		Slot<int32_t> o_undrained;
		Slot<uint8_t *> o_state;
		Slot<uint16_t> o_head;
		Slot<uint2> o_cut; // open runs: per stream (covered, SetInput call) of the last cut, (0, 0) for none
	} fast;
	struct { // level 0 (stored_layout)
		b200z_stored_state *state = nullptr; // caller's host array, used while the plan is built
		int n_blocks = 0;
		Slot<StoredBlock> o_blocks;
		Slot<int64_t> o_lens;
		std::vector<uint2> cut; // open runs: the same as fast.o_cut, known when the plan is built
	} stored;
};

static int64_t hist_len(const DeflatePlan *p, int i) { return p->hist.empty() ? 0 : p->hist[i]; }

// levels 1-9: room for each stream's symbols and for the most blocks they can be cut into
static void blocks_layout(DeflatePlan *p) {
	const int n = p->n;
	std::vector<uint32_t> blk_off(n + 1);
	std::vector<int32_t> blk_desc;
	uint32_t nblk = 0;
	for (int i = 0; i < n; i++) {
		blk_off[i] = nblk;
		const uint32_t maxb = (uint32_t)(p->in_len[i] / kBlockSyms) + 2;
		blk_desc.insert(blk_desc.end(), maxb, i);
		nblk += maxb;
	}
	blk_off[n] = nblk;
	p->n_blkmax = (int)nblk;
	Arena &ws = p->ws;
	p->o_sym = ws.reserve<uint32_t>(p->in_bytes + 16);
	p->o_blk_desc = ws.upload(blk_desc, 1);
	p->o_blk_off = ws.upload(blk_off);
	p->o_nsyms = ws.reserve<uint32_t>(n);
	p->o_nblocks = ws.reserve<uint32_t>(n);
	p->o_blk_start = ws.reserve<uint32_t>(nblk + 1);
	p->o_blk_ptop = ws.reserve<uint32_t>(nblk + 1);
	p->o_meta = ws.reserve<BlockMeta>(nblk + 1);
	p->o_tables = ws.reserve<BlockTables>(nblk + 1);
}

// levels 5-9
static void lazy_layout(DeflatePlan *p, int64_t maxlen, int sms) {
	auto &z = p->lazy;
	const int n = p->n;
	// chunk of the parse: 32 Ki positions (one warp each); k_parse_fix only compares states at their boundaries, so a long
	// stream may have tens of thousands of them (grown beyond 65536 chunks per stream)
	uint32_t chunk = 32768;
	{
		const int64_t need = (maxlen / 65536 + kRound - 1) / kRound * kRound;
		if (need > (int64_t)chunk) chunk = (uint32_t)need;
	}
	z.parse_chunk = chunk;
	// Run length of k_links (a multiple of 32768, 65536 .. 1048576).  Every run but a stream's first re-walks 32768 positions
	// to warm its head table up (37 % more steps than positions with 64 Ki runs on 256 KiB buffers, 12 % with 128 Ki runs,
	// none with 256 Ki runs), while fewer, longer CTAs fill the last wave worse (three CTAs fit an SM).  The plan takes the
	// length with the smallest estimate of waves x steps per run; B200Z_LINK_RUN=<positions> overrides it for timing.
	z.link_run = kRun;
	{
		const int64_t slots = 3ll * sms;
		double best = 0;
		for (int64_t run = 65536; run <= 1048576; run *= 2) {
			int64_t ctas = 0, longest = 0;
			for (int i = 0; i < n; i++) {
				const int64_t len = p->in_len[i];
				ctas += (len + run - 1) / run;
				const int64_t first = len < run ? len : run;
				const int64_t steps = len > run ? run + 32768 : first; // a run behind the first also walks its warm-up
				longest = steps > longest ? steps : longest;
			}
			const double est = (double)((ctas + slots - 1) / slots) * (double)longest;
			if (best == 0 || est < best * 0.97) { // (a longer run has to win clearly: its CTAs are the less balanced ones)
				best = est;
				z.link_run = (int)run;
			}
			if (run >= maxlen) break;
		}
	}
	if (const char *e = getenv("B200Z_LINK_RUN")) {
		const long v = atol(e);
		if (v >= 65536 && v <= 1048576 && v % 32768 == 0) z.link_run = (int)v;
	}
	std::vector<int2> runs, tiles, rgroups;
	std::vector<ChunkDesc> chunks;
	std::vector<uint32_t> rnd_off(n + 1);
	std::vector<int64_t> hm_off(n, 0);
	std::vector<uint8_t> hmask;
	uint32_t nrounds = 0;
	z.entry.resize(n);
	for (int i = 0; i < n; i++) {
		const int64_t len = p->in_len[i], H = hist_len(p, i);
		for (int64_t s = 0; s < len; s += z.link_run) runs.push_back(make_int2(i, (int)s));
		for (int64_t s = 0; s < len; s += kTile) tiles.push_back(make_int2(i, (int)s));
		for (int64_t s = 0; s < len; s += chunk)
			chunks.push_back(ChunkDesc{i, (uint32_t)s, (uint32_t)(len - s > (int64_t)chunk ? s + chunk : len)});
		rnd_off[i] = nrounds;
		const uint32_t nr = (uint32_t)((len + kRound - 1) / kRound);
		for (uint32_t r = 0; r < nr; r += 4) rgroups.push_back(make_int2(i, (int)r));
		nrounds += nr;
		z.entry[i] = RoundRec{(uint32_t)H, (uint32_t)kMinMatch - 1, 0u, 0u, (uint32_t)H, 0u};
		if (!p->hist.empty()) {
			hm_off[i] = (int64_t)hmask.size();
			hmask.resize(hmask.size() + (size_t)H + 1, 0);
			uint8_t *m = hmask.data() + hm_off[i];
			if (!z.hist_mask[i].empty()) memcpy(m, z.hist_mask[i].data(), (size_t)H);
			else if (H) m[H - 1] = 1, m[H > 1 ? H - 2 : 0] = 1; // the last two positions of a dictionary/segment are never inserted
		}
	}
	rnd_off[n] = nrounds;
	z.n_runs = (int)runs.size();
	z.n_tiles = (int)tiles.size();
	z.n_chunks = (int)chunks.size();
	z.n_rgroups = (int)rgroups.size();
	Arena &ws = p->ws;
	const int64_t io = p->in_bytes;
	z.o_run_desc = ws.upload(runs, 1);
	z.o_tile_desc = ws.upload(tiles, 1);
	z.o_hm_off = ws.upload(hm_off, 1);
	z.o_hmask = ws.upload(hmask, 16);
	z.o_link = ws.reserve<uint16_t>(io + 32);
	z.o_mt = ws.reserve<uint2>(io + 8);
	z.o_sym_local = ws.reserve<uint32_t>(io + 16);
	z.o_chunks = ws.upload(chunks, 1);
	z.o_rgroups = ws.upload(rgroups, 1);
	z.o_rnd_off = ws.upload(rnd_off);
	z.o_recs = ws.reserve<RoundRec>(nrounds + 1);
	z.o_ents = ws.reserve<RoundRec>(nrounds + 1);
	z.o_rnd_symoff = ws.reserve<uint32_t>(nrounds + 1);
	z.o_entry = ws.upload(z.entry, 1);
	z.o_cut = ws.reserve<RoundRec>(n + 1);
	blocks_layout(p);
	// lazy_launch: k_links, k_match, k_parse_chunk, k_parse_fix, k_parse_scan, k_parse_gather (+ k_parse_cut for an open
	// run), then k_plan, k_scan, k_emit
	p->launches = 9 + (p->end_mode == B200Z_END_NONE ? 1 : 0);
}

// stages: B200Z_STAGE_SEARCH = match finding (k_links, k_match), B200Z_STAGE_ENCODE = the parse
static int lazy_launch(DeflatePlan *p, const uint8_t *d_in, cudaStream_t s, bool do_search, bool do_encode) {
	const auto &z = p->lazy;
	const Arena &ws = p->ws;
	const int n = p->n;
	const LevelParams lp = level_params(p->level);
	const int64_t *in_off = ws.at(p->o_in_off), *in_len = ws.at(p->o_in_len);
	uint16_t *link = ws.at(z.o_link);
	uint2 *mt = ws.at(z.o_mt);
	uint32_t *sym = ws.at(p->o_sym);
	const uint32_t *hist = ws.at(p->o_hist);
	const int64_t *bias = ws.at(p->o_bias);
	if (do_search) {
		p->mark(s, "k_links");
		if (z.n_runs)
			k_links<<<z.n_runs, kLinkThreads, kLinksSmem, s>>>(d_in, link, in_off, in_len, ws.at(z.o_run_desc), hist,
			                                                   ws.at(z.o_hmask), ws.at(z.o_hm_off), (uint32_t)z.link_run);
		p->mark(s, "k_match");
		if (z.n_tiles)
			k_match<<<z.n_tiles, kMatchThreads, kTileData + 2 * 2 * kTile, s>>>(d_in, link, mt, in_off, in_len,
			                                                                   ws.at(z.o_tile_desc), hist, bias, sym, lp);
	}
	if (!do_encode) return B200Z_OK;
	p->mark(s, "k_parse");
	uint32_t *sym_local = ws.at(z.o_sym_local);
	const uint32_t *rnd_off = ws.at(z.o_rnd_off);
	RoundRec *recs = ws.at(z.o_recs), *ents = ws.at(z.o_ents);
	uint32_t *rnd_symoff = ws.at(z.o_rnd_symoff);
	uint32_t *nsyms = ws.at(p->o_nsyms), *nblocks = ws.at(p->o_nblocks), *blk_off = ws.at(p->o_blk_off);
	uint32_t *blk_start = ws.at(p->o_blk_start), *blk_ptop = ws.at(p->o_blk_ptop);
	if (z.n_chunks)
		k_parse_chunk<<<z.n_chunks, 32, kParseSmem, s>>>(d_in, link, mt, sym_local, in_off, in_len, ws.at(z.o_chunks), rnd_off,
		                                                 recs, ents, hist, bias, ws.at(z.o_entry), lp, p->strategy, parse_warm(),
		                                                 p->end_mode);
	k_parse_fix<<<n, 32, kParseSmem, s>>>(d_in, link, mt, sym_local, in_off, in_len, rnd_off, recs, ents, z.parse_chunk, hist,
	                                      bias, lp, p->strategy, p->end_mode);
	k_parse_scan<<<n, 256, 0, s>>>(d_in, in_off, in_len, rnd_off, recs, rnd_symoff, sym, nsyms, nblocks, blk_off, blk_start,
	                               blk_ptop, hist, p->end_mode);
	if (z.n_rgroups)
		k_parse_gather<<<z.n_rgroups, 128, 0, s>>>(sym_local, sym, in_off, in_len, ws.at(z.o_rgroups), rnd_off, recs,
		                                           rnd_symoff, blk_off, blk_start, blk_ptop, hist);
	if (p->end_mode == B200Z_END_NONE)
		k_parse_cut<<<(n + 127) / 128, 128, 0, s>>>(d_in, link, mt, in_off, in_len, rnd_off, recs, rnd_symoff, nblocks, bias,
		                                            ws.at(z.o_entry), ws.at(z.o_cut), n, lp, p->strategy);
	return B200Z_OK;
}

// levels 1-4
static void fast_layout(DeflatePlan *p, int64_t maxlen, int sms) {
	auto &f = p->fast;
	const int n = p->n;
	// size of k_fast's prev[] table (see there)
	const int64_t need = maxlen + 2;
	f.prev_entries = 32768;
	if (need <= 32768 && f.engine_state.empty()) f.prev_entries = (int)((need + 255) / 256 * 256); // (a carried state holds whole tables)
	// persistent one-warp CTAs: as many per SM as their prev[] tables fit (head[] is in the pool), 16 at most
	int per_sm = (int)((227 * 1024) / (2 * f.prev_entries + 1024));
	if (per_sm > 16) per_sm = 16;
	if (per_sm < 1) per_sm = 1;
	const int64_t slots = (int64_t)sms * per_sm;
	f.ctas = (int)(n < slots ? n : slots);
	f.head_smem = n <= sms; // nothing to gain from sharing SMs: keep head[] next to prev[] (k_fast)
	if (const char *e = getenv("B200Z_FAST_HEAD")) f.head_smem = e[0] == 's'; // "smem" / "pool": for tests and timing
	Arena &ws = p->ws;
	f.o_sched = ws.upload(p->sched, 1);
	f.o_sched_off = ws.upload(p->sched_off);
	f.o_undrained = ws.upload(p->undrained, 1);
	f.o_state = ws.upload(f.engine_state.empty() ? std::vector<uint8_t *>(n) : f.engine_state, 1);
	f.o_head = ws.reserve<uint16_t>(f.head_smem ? 128 : 32768ll * f.ctas);
	f.o_counter = ws.reserve<uint32_t>(64);
	f.o_cut = ws.reserve<uint2>(n + 1);
	blocks_layout(p);
	p->launches = 4; // k_fast, then k_plan, k_scan, k_emit (the memset of the CTA counter is not counted)
}

static int fast_launch(DeflatePlan *p, const uint8_t *d_in, cudaStream_t s) {
	const auto &f = p->fast;
	const Arena &ws = p->ws;
	p->mark(s, "k_fast");
	B200Z_CUDA(cudaMemsetAsync(ws.at(f.o_counter), 0, 4, s));
	k_fast<<<f.ctas, 32, 2 * f.prev_entries + (f.head_smem ? 65536 : 0), s>>>(
	    d_in, ws.at(p->o_sym), ws.at(p->o_in_off), ws.at(p->o_in_len), ws.at(p->o_nsyms), ws.at(p->o_nblocks), ws.at(p->o_blk_off),
	    ws.at(p->o_blk_start), ws.at(p->o_blk_ptop), ws.at(p->o_hist), level_params(p->level), p->strategy, p->end_mode,
	    f.prev_entries, ws.at(f.o_sched), ws.at(f.o_sched_off), ws.at(f.o_undrained), ws.at(f.o_state),
	    p->hist_kind == B200Z_HIST_CONTINUE ? 1 : 0, fast_group_enabled(), p->n, f.head_smem ? nullptr : ws.at(f.o_head),
	    ws.at(f.o_counter), ws.at(f.o_cut));
	return B200Z_OK;
}

// level 0: the blocks DeflateStored writes follow from the lengths and the schedule alone.  Lowers ck_len to the bytes each
// stream's window took in, and writes the state behind the run back to stored.state.
static void stored_layout(DeflatePlan *p, std::vector<int64_t> &ck_len) {
	auto &st = p->stored;
	const int n = p->n;
	const bool cont = p->hist_kind == B200Z_HIST_CONTINUE;
	std::vector<StoredBlock> blocks;
	std::vector<int64_t> lens;
	for (int i = 0; i < n; i++) {
		const int64_t len = p->in_len[i], H = hist_len(p, i);
		uint64_t dst = 0;
		const int nch = (int)(p->sched_off[i + 1] - p->sched_off[i]);
		const uint32_t *cum = nch ? p->sched.data() + p->sched_off[i] : nullptr;
		const bool busy_last = !p->undrained[i];
		StoredCarry cin{0, 0, 0, 0}, cout{0, 0, 0, 0};
		if (cont) // checked when the plan was created: stored.state is there
			cin = StoredCarry{st.state[i].strstart, st.state[i].block_start, st.state[i].slides, st.state[i].input_off};
		// (the carried state fixes where the data starts: pos_base is not needed, and may have any size)
		const uint32_t start_bias = cont ? stored_rebase(cin, (uint32_t)H) : 0u;
		int cut_call = 0;
		stored_run((uint32_t)(len - H), cont ? 0u : (uint32_t)H, p->end_mode, [&](uint32_t start, uint32_t blen, bool last) {
			blocks.push_back(StoredBlock{i, start, blen, last ? 1u : 0u, dst});
			dst += 5 + (uint64_t)blen;
		}, cum, nch, cont ? &cin : nullptr, &cout, start_bias, busy_last, &cut_call);
		if (p->end_mode == B200Z_END_NONE) // the data in front of the last block's end; none written: the entry state
			st.cut.push_back(make_uint2(blocks.empty() || blocks.back().stream != i ? 0u
			                                                   : blocks.back().src + blocks.back().len - (uint32_t)H,
			                            (uint32_t)cut_call));
		// what the window took in: everything, except when Finish() right behind an undrained SetInput makes
		// DeflateStored end the stream early (lastBlock = finish although input is left, DeflaterEngine.cs:629-641);
		// TotalIn and the Adler-32 of the reference then cover the consumed bytes only, and so do ours.  (Behind the
		// cut of an open run the data starts strstart - blockStart bytes in front of inputOff.)
		const int64_t taken = (int64_t)(uint32_t)(cout.inputOff - (cont ? cin.inputOff - (uint32_t)(cin.strstart - cin.blockStart) : 0u));
		if (taken < ck_len[i]) ck_len[i] = taken;
		if (st.state) st.state[i] = b200z_stored_state{cout.strstart, cout.blockStart, cout.slides, cout.inputOff}; // (behind an open run: the state at its cut)
		lens.push_back((int64_t)dst);
	}
	st.n_blocks = (int)blocks.size();
	st.o_blocks = p->ws.upload(blocks, 1);
	st.o_lens = p->ws.upload(lens, 1);
	p->launches = 2; // k_stored, k_set_results
}

static void stored_launch(DeflatePlan *p, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                          int64_t *d_out_bits, cudaStream_t s) {
	const auto &st = p->stored;
	const Arena &ws = p->ws;
	p->mark(s, "k_stored");
	if (st.n_blocks) k_stored<<<st.n_blocks, 256, 0, s>>>(d_in, d_out, ws.at(p->o_in_off), ws.at(p->o_out_off), ws.at(st.o_blocks));
	k_set_results<<<(p->n + 127) / 128, 128, 0, s>>>(p->n, ws.at(st.o_lens), d_out_len, d_status, d_out_bits);
}

static int deflate_plan_build(DeflatePlan *p) {
	const int n = p->n;
	p->in_off.resize(n);
	p->out_off.resize(n);
	p->out_cap.resize(n);
	std::vector<uint32_t> hist32(n);
	std::vector<int64_t> ck_off(n), ck_len(n);
	int64_t io = 0, oo = 0, maxlen = 0;
	for (int i = 0; i < n; i++) {
		const int64_t len = p->in_len[i], H = hist_len(p, i);
		if (len < 0 || len > 0xFFFF0000ll) {
			set_error("stream %d: length %lld out of range", i, (long long)len);
			return B200Z_E_ARG;
		}
		hist32[i] = (uint32_t)H;
		p->in_off[i] = io;
		io += align_up(len + 16, kAlign);
		p->out_off[i] = oo;
		p->out_cap[i] = align_up(b200z_deflate_bound(len), kAlign);
		oo += p->out_cap[i];
		ck_off[i] = p->in_off[i] + H; // the checksum covers the data, never the history
		ck_len[i] = len - H;
		maxlen = len > maxlen ? len : maxlen;
	}
	p->in_bytes = io;
	p->out_bytes = oo;
	Arena &ws = p->ws;
	p->upload_streams(p->in_off, p->in_len, 0);
	p->o_hist = ws.upload(hist32, 1);
	p->o_bias = ws.upload(p->bias, 1);
	p->o_bitbase = ws.upload(p->bit_base, 1);
	int sms = 0;
	if (sm_count(&sms) != cudaSuccess) sms = 132;
	switch (level_params(p->level).func) {
	case 0: stored_layout(p, ck_len); break;
	case 1: fast_layout(p, maxlen, sms); break;
	default: lazy_layout(p, maxlen, sms);
	}
	if (p->wrap != B200Z_WRAP_RAW) {
		p->o_ck_off = ws.upload(ck_off, 1);
		p->o_ck_len = ws.upload(ck_len, 1);
		std::vector<CkTile> ck_tiles;
		checksum_tiles(ck_len.data(), n, ck_tiles, p->wrap == B200Z_WRAP_ZLIB ? 1 : 0);
		p->n_ck_tiles = (int)ck_tiles.size();
		p->o_ck_desc = ws.upload(ck_tiles, 1);
		p->o_ck_acc = ws.reserve<unsigned long long>(2ll * (n + 1));
		if (p->end_mode != B200Z_END_NONE) p->launches += 3; // checksum_launch (deflate_plan_run)
	}
	int rc = ws.alloc();
	if (rc) return rc;
	B200Z_CUDA(cudaFuncSetAttribute(k_fast, cudaFuncAttributeMaxDynamicSharedMemorySize, kFastSmem));
	B200Z_CUDA(cudaFuncSetAttribute(k_links, cudaFuncAttributeMaxDynamicSharedMemorySize, kLinksSmem));
	B200Z_CUDA(cudaFuncSetAttribute(k_match, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileData + 2 * 2 * kTile));
	B200Z_CUDA(cudaFuncSetAttribute(k_plan, cudaFuncAttributePreferredSharedMemoryCarveout, 100)); // 24 CTAs per SM
	return B200Z_OK;
}

int deflate_plan_create(int32_t n, const int64_t *in_len, int level, int strategy, int wrap, int end_mode,
                        const b200z_history *hist, b200z_plan **out) {
	std::unique_ptr<DeflatePlan> p(new DeflatePlan());
	p->device = current_device();
	p->kind = 0;
	p->n = n;
	p->level = level;
	p->strategy = strategy;
	p->wrap = wrap;
	p->end_mode = end_mode;
	p->in_len.assign(in_len, in_len + n);
	static const b200z_history no_history{}; // (all NULL: what a plan without history reads)
	if (!hist || n == 0) hist = &no_history;
	const int kind = hist->kind;
	if (level <= 4 && (end_mode == B200Z_END_NONE || kind == B200Z_HIST_CONTINUE)) {
		// DeflateStored / DeflateFast keep window-relative tables across Deflate() calls that depend on the parse, not on the
		// stream position: a stream that goes on after Flush() reads them from the run of the previous segment, and the cut
		// of an open run writes them for the next one
		bool have = (level == 0 ? hist->stored_state != nullptr : hist->engine_state != nullptr);
		for (int i = 0; have && level >= 1 && i < n; i++) have = hist->engine_state[i] != nullptr;
		if (!have) {
			set_error("continuing a stream after Flush() and open runs (B200Z_END_NONE) at levels 0-4 need the engine state "
			          "(b200z_history.engine_state / stored_state)");
			return B200Z_E_UNSUPPORTED;
		}
	}
	// levels 0-4: the call pattern and the engine state between segments (header: "streams with history")
	const bool sched = level <= 4 && hist->chunk_count;
	if (sched && !hist->chunk_len) {
		set_error("history: chunk_count without chunk_len");
		return B200Z_E_ARG;
	}
	if (kind != B200Z_HIST_NONE && ((kind != B200Z_HIST_DICTIONARY && kind != B200Z_HIST_CONTINUE) || !hist->hist_len)) {
		set_error("history: kind/hist_len");
		return B200Z_E_ARG;
	}
	p->hist_kind = kind;
	p->check_seeded = kind != B200Z_HIST_NONE && hist->check_seeded != 0;
	if (kind != B200Z_HIST_NONE) p->hist.assign(hist->hist_len, hist->hist_len + n);
	p->bias.assign(n, 0);
	p->bit_base.assign(n, 0u);
	p->lazy.hist_mask.resize(n);
	p->sched_off.assign(n + 1, 0u);
	p->undrained.assign(n, 0);
	if (hist->engine_state) p->fast.engine_state.resize(n);
	p->stored.state = hist->stored_state;
	for (int i = 0; i < n; i++) {
		if (sched) {
			int64_t sum = 0;
			for (int k = 0; k < hist->chunk_count[i]; k++) {
				const int64_t c = hist->chunk_len[i] ? hist->chunk_len[i][k] : -1;
				if (c < 0) {
					set_error("stream %d: SetInput size %d", i, k);
					return B200Z_E_ARG;
				}
				sum += c;
				p->sched.push_back((uint32_t)sum);
			}
			if (hist->chunk_count[i] < 0 || (hist->chunk_count[i] > 0 && sum != in_len[i])) {
				set_error("stream %d: the SetInput sizes add up to %lld, the stream has %lld bytes", i, (long long)sum,
				          (long long)in_len[i]);
				return B200Z_E_ARG;
			}
		}
		p->sched_off[i + 1] = (uint32_t)p->sched.size();
		p->undrained[i] = hist->undrained_last && hist->undrained_last[i] ? 1 : 0;
		if (hist->engine_state) p->fast.engine_state[i] = static_cast<uint8_t *>(hist->engine_state[i]);
		if (kind == B200Z_HIST_NONE) continue;
		const int64_t H = p->hist[i];
		if (H < 0 || H > 32768 || (kind == B200Z_HIST_DICTIONARY && H > kMaxDist)) {
			set_error("stream %d: history of %lld bytes (at most %d)", i, (long long)H, kind == B200Z_HIST_DICTIONARY ? kMaxDist : 32768);
			return B200Z_E_ARG;
		}
		int64_t pos_base = (hist->pos_base && kind == B200Z_HIST_CONTINUE) ? hist->pos_base[i] : H;
		const int32_t bit_base = hist->bit_base ? hist->bit_base[i] : 0;
		// (levels 0-4 keep positions relative to the carried engine state: carry_rebase)
		if (pos_base < H || bit_base < 0 || bit_base > 7) {
			set_error("stream %d: pos_base/bit_base", i);
			return B200Z_E_ARG;
		}
		// Levels 5-9 read the position only through the window phase, which is periodic with 32768 from kSlideFirst on
		// (is_slide_pos, slides_done; storedOffset moves with both): the equal phase in the first period keeps the
		// kernels' 32-bit positions valid in a stream of any length
		if (level >= 5 && pos_base >= (int64_t)kSlideFirst) pos_base = (int64_t)kSlideFirst + (pos_base - (int64_t)kSlideFirst) % 32768;
		if (level >= 5 && pos_base + in_len[i] > 0xFFFFFFFFll) {
			set_error("stream %d: %lld bytes behind position %lld do not fit one plan slot", i, (long long)in_len[i],
			          (long long)pos_base);
			return B200Z_E_ARG;
		}
		p->bias[i] = pos_base - H;
		p->bit_base[i] = (uint32_t)bit_base;
		if (hist->hist_mask && hist->hist_mask[i]) p->lazy.hist_mask[i].assign(hist->hist_mask[i], hist->hist_mask[i] + H);
		p->in_len[i] += H; // the input slot holds history + data
	}
	const int rc = deflate_plan_build(p.get());
	if (rc == B200Z_OK) *out = p.release();
	return rc;
}

int deflate_plan_run(b200z_plan *plan, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                     uint32_t *d_check, int64_t *d_out_bits, cudaStream_t s, int stages) {
	DeflatePlan *p = static_cast<DeflatePlan *>(plan);
	const Arena &ws = p->ws;
	const int n = p->n;
	if (n == 0) return B200Z_OK;
	const int func = level_params(p->level).func;
	// stages: B200Z_STAGE_SEARCH = match finding (levels 5-9: k_links, k_match), B200Z_STAGE_ENCODE = everything else.
	// Splitting lets a caller put other work (e.g. an inflate plan on a second stream) next to the ENCODE kernels, which
	// leave most of an SM's shared memory free, instead of next to k_match, which takes all of it.
	const bool do_search = (stages & B200Z_STAGE_SEARCH) != 0, do_encode = (stages & B200Z_STAGE_ENCODE) != 0;
	const bool was_timing = p->timing;
	if (stages != (B200Z_STAGE_SEARCH | B200Z_STAGE_ENCODE)) p->timing = false; // per-kernel times are for whole runs
	struct TimingRestore {
		b200z_plan *p;
		bool v;
		~TimingRestore() { p->timing = v; }
	} timing_restore{p, was_timing};
	if (func != 2 && !do_encode) return B200Z_OK; // levels 0-4 have no separate search stage
	p->ev_used = 0;
	if (func == 0) {
		stored_launch(p, d_in, d_out, d_out_len, d_status, d_out_bits, s);
	} else {
		if (do_encode) {
			p->mark(s, "memset");
			B200Z_CUDA(cudaMemsetAsync(d_out, 0, (size_t)p->out_bytes, s));
		}
		const int rc = func == 1 ? fast_launch(p, d_in, s) : lazy_launch(p, d_in, s, do_search, do_encode);
		if (rc) return rc;
		if (!do_encode) {
			B200Z_CUDA(cudaGetLastError());
			return B200Z_OK;
		}
		// Huffman trees per block, block offsets, the bits
		const int64_t *in_off = ws.at(p->o_in_off), *out_off = ws.at(p->o_out_off);
		uint32_t *sym = ws.at(p->o_sym), *nblocks = ws.at(p->o_nblocks), *blk_off = ws.at(p->o_blk_off);
		int32_t *blk_desc = ws.at(p->o_blk_desc);
		BlockMeta *meta = ws.at(p->o_meta);
		BlockTables *tables = ws.at(p->o_tables);
		p->mark(s, "k_plan");
		k_plan<<<p->n_blkmax, kPlanThreads, 0, s>>>(sym, in_off, ws.at(p->o_in_len), ws.at(p->o_nsyms), nblocks, blk_off, blk_desc,
		                                            ws.at(p->o_blk_start), ws.at(p->o_blk_ptop), meta, tables, ws.at(p->o_bias),
		                                            p->end_mode);
		p->mark(s, "k_scan");
		k_scan<<<(n + 127) / 128, 128, 0, s>>>(n, nblocks, blk_off, meta, d_out, out_off, ws.at(p->o_out_cap), d_out_len, d_status,
		                                       d_out_bits, ws.at(p->o_bitbase), p->end_mode);
		p->mark(s, "k_emit");
		k_emit<<<p->n_blkmax, 256, 0, s>>>(d_in, sym, d_out, in_off, out_off, nblocks, blk_off, blk_desc, meta, tables);
	}
	p->mark(s, "checksum");
	// (an open run leaves the running checksum alone: its caller knows which of the bytes the run covered)
	if (p->end_mode == B200Z_END_NONE) {
		p->cut_ready = true;
	} else if (p->wrap != B200Z_WRAP_RAW && d_check) {
		int rc = checksum_launch(p->wrap == B200Z_WRAP_ZLIB ? 1 : 0, d_in, ws.at(p->o_ck_off), ws.at(p->o_ck_len), n,
		                         ws.at(p->o_ck_desc), p->n_ck_tiles, ws.at(p->o_ck_acc), d_check, p->check_seeded ? 0 : 1, s, false);
		if (rc) return rc;
	}
	p->mark(s, "end");
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

int deflate_plan_set_entry(b200z_plan *plan, const b200z_parse_entry *entry) {
	DeflatePlan *p = static_cast<DeflatePlan *>(plan);
	if (p->level < 5) {
		set_error("entry states are for levels 5-9");
		return B200Z_E_UNSUPPORTED;
	}
	std::vector<RoundRec> v(p->lazy.entry);
	for (int i = 0; i < p->n; i++) {
		const b200z_parse_entry &e = entry[i];
		const int64_t H = hist_len(p, i);
		const int64_t data = p->in_len[i] - H;
		const bool pending = e.match_len >= kMinMatch;
		// with nothing pending matchLen is MIN_MATCH - 1; a byte left pending lies in the data, and so does its match
		if (e.prev_available < 0 || e.prev_available > 1 || e.match_len < kMinMatch - 1 || e.match_len > kMaxMatch ||
		    (pending && (!e.prev_available || e.match_dist < 1 || e.match_dist > kMaxDist || e.match_dist > H)) ||
		    (!pending && e.match_dist != 0) || (e.prev_available && data < (pending ? e.match_len : 1))) {
			set_error("stream %d: entry state (prev_available %d, match_len %d, match_dist %lld) with %lld history and %lld data bytes",
			          i, e.prev_available, e.match_len, (long long)e.match_dist, (long long)H, (long long)data);
			return B200Z_E_ARG;
		}
		v[i].p = (uint32_t)(H + e.prev_available);
		v[i].mlen = (uint32_t)e.match_len;
		v[i].mstart = pending ? (uint32_t)(H - e.match_dist) : 0u;
		v[i].prevAvail = (uint32_t)e.prev_available;
	}
	const int rc = p->ws.write(p->lazy.o_entry, v);
	if (rc == B200Z_OK) p->lazy.entry = v;
	return rc;
}

// levels 0-4: per stream (covered, SetInput call) of the last cut
static int fast_cuts(DeflatePlan *p, std::vector<uint2> &v, cudaStream_t s) {
	if (p->level == 0) {
		v = p->stored.cut;
		return B200Z_OK;
	}
	v.resize((size_t)p->n);
	B200Z_CUDA(cudaMemcpyAsync(v.data(), p->ws.at(p->fast.o_cut), sizeof(uint2) * v.size(), cudaMemcpyDeviceToHost, s));
	B200Z_CUDA(cudaStreamSynchronize(s));
	return B200Z_OK;
}

int deflate_plan_get_cut(b200z_plan *plan, int64_t *covered, b200z_parse_entry *next, cudaStream_t s) {
	DeflatePlan *p = static_cast<DeflatePlan *>(plan);
	if (p->end_mode != B200Z_END_NONE || !p->cut_ready) {
		set_error("a cut is reported after a run of a B200Z_END_NONE plan");
		return B200Z_E_STATE;
	}
	if (p->level <= 4) { // the engine state at the cut is in engine_state / stored_state; nothing is pending
		std::vector<uint2> v;
		const int rc = fast_cuts(p, v, s);
		if (rc) return rc;
		for (int i = 0; i < p->n; i++) {
			covered[i] = v[i].x;
			if (next) next[i] = b200z_parse_entry{0, kMinMatch - 1, 0};
		}
		return B200Z_OK;
	}
	std::vector<RoundRec> v((size_t)p->n);
	B200Z_CUDA(cudaMemcpyAsync(v.data(), p->ws.at(p->lazy.o_cut), sizeof(RoundRec) * v.size(), cudaMemcpyDeviceToHost, s));
	B200Z_CUDA(cudaStreamSynchronize(s));
	for (int i = 0; i < p->n; i++) {
		const int64_t H = hist_len(p, i);
		const int64_t pos = (int64_t)v[i].p - v[i].prevAvail; // the first byte not written
		covered[i] = pos - H;
		next[i].prev_available = (int32_t)v[i].prevAvail;
		next[i].match_len = (int32_t)v[i].mlen;
		next[i].match_dist = v[i].mlen >= (uint32_t)kMinMatch ? pos - (int64_t)v[i].mstart : 0;
	}
	return B200Z_OK;
}

int deflate_plan_get_cut_call(b200z_plan *plan, int32_t *call, cudaStream_t s) {
	DeflatePlan *p = static_cast<DeflatePlan *>(plan);
	if (p->end_mode != B200Z_END_NONE || !p->cut_ready || p->level > 4) {
		set_error("a cut's SetInput call is reported after a run of a level 0-4 B200Z_END_NONE plan");
		return B200Z_E_STATE;
	}
	std::vector<uint2> v;
	const int rc = fast_cuts(p, v, s);
	if (rc) return rc;
	for (int i = 0; i < p->n; i++) call[i] = (int32_t)v[i].y;
	return B200Z_OK;
}

} // namespace b200z
