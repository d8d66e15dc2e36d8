// b200z_core.cuh -- per-thread building blocks of the H100 DEFLATE engine.
//
// Everything here is a __host__ __device__ inline function so that the same code that runs
// inside the sm_90a kernels can be executed serially by tests/cpu_model (a g++-compiled harness
// that checks the *parallel decomposition* -- link table, per-position match table, parse state
// machine, block planner, tree builder, bit emitter -- against the oracle without a GPU).
//
// The decomposition (DESIGN.md "Deflate pipeline"), for the reference's lazy levels 5-9
// (DeflaterEngine.DeflateSlow, DeflaterEngine.cs:741-855):
//   K1 links   : link[p] = distance to the previous position with the same 15-bit hash
//                (what head[]/prev[] of DeflaterEngine.InsertString :417-439 encode; in slow mode every
//                position is inserted, so the chains are a pure function of the bytes)
//   K2 matches : for EVERY position the result FindLongestMatch (:474-612) would return when entered
//                with matchLen < goodLength (full chain budget, "A") and with matchLen >= goodLength
//                (quartered budget, "B"), both from threshold 2; any other incoming threshold m0 < nice
//                only filters that result (len > m0), see parse_step().
//   K3 parse   : the sequential lazy-evaluation state machine (prevAvailable, matchLen, matchStart)
//   K4 plan    : per 16384-symbol block: histograms, the reference's bespoke Huffman construction
//                (DeflaterHuffman.Tree.BuildTree/BuildLength/BuildCodes :196-329, :475-579, :151-194),
//                block type decision and exact bit size (FlushBlock :788-857)
//   K5 scan    : bit offset of every block inside its stream
//   K6 emit    : header + per-symbol codes at prefix-summed bit offsets
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define B200Z_HD __host__ __device__ __forceinline__
#define B200Z_HDN __host__ __device__ inline
#else
#define B200Z_HD inline
#define B200Z_HDN inline
#endif

namespace b200z {

// ---- DeflaterConstants.cs ------------------------------------------------------------------
constexpr int kMaxMatch = 258;
constexpr int kMinMatch = 3;
constexpr int kWSize = 32768;
constexpr int kMaxDist = kWSize - (kMaxMatch + kMinMatch + 1); // 32506, DeflaterConstants.cs:94
constexpr int kTooFar = 4096;                                  // DeflaterEngine.cs:51
constexpr int kBlockSyms = 16384;                              // DeflaterHuffman.BUFSIZE, DeflaterHuffman.cs:15
constexpr int kLiteralNum = 286, kDistNum = 30, kBitlenNum = 19;
// build_tree's scratch for a tree of n symbols (18 * n + 3 bytes, see there), and for the literal tree
B200Z_HD constexpr int tree_scratch_ints(int n) { return (9 * n + 3) / 2 + 2; }
constexpr int kTreeScratchInts = tree_scratch_ints(kLiteralNum);
constexpr int kHdrWords = 160; // dynamic header: <= 17 + 57 + 316 * 14 bits = 4498 bits < 160 * 32
constexpr uint32_t kSlideFirst = 65273; // first input offset whose window index reaches 65274 (trap T8)

struct LevelParams {
	int good, lazy, nice, chain, func;
};

constexpr int kLevelChain[10] = {0, 4, 8, 32, 16, 32, 128, 256, 1024, 4096}; // MAX_CHAIN, DeflaterConstants.cs:139
// k_match tests the budgets of levels 5-9 (chain and chain >> 2) once per four candidates
static_assert(kLevelChain[5] % 16 == 0 && kLevelChain[6] % 16 == 0 && kLevelChain[7] % 16 == 0 && kLevelChain[8] % 16 == 0 &&
                  kLevelChain[9] % 16 == 0,
              "level 5-9 chain budgets must be multiples of 16");

B200Z_HD LevelParams level_params(int level) { // DeflaterConstants.cs:124-144
	const int good[10] = {0, 4, 4, 4, 4, 8, 8, 8, 32, 32};
	const int lazy[10] = {0, 4, 5, 6, 4, 16, 16, 32, 128, 258};
	const int nice[10] = {0, 8, 16, 32, 16, 32, 128, 128, 258, 258};
	const int func[10] = {0, 1, 1, 1, 1, 2, 2, 2, 2, 2};
	LevelParams lp;
	lp.good = good[level];
	lp.lazy = lazy[level];
	lp.nice = nice[level];
	const int chain[10] = {kLevelChain[0], kLevelChain[1], kLevelChain[2], kLevelChain[3], kLevelChain[4],
	                       kLevelChain[5], kLevelChain[6], kLevelChain[7], kLevelChain[8], kLevelChain[9]}; // constant indices: usable on the device
	lp.chain = chain[level];
	lp.func = func[level];
	return lp;
}

// 15-bit hash of 3 bytes: the closed form of UpdateHash/InsertString's rolling value
// (DeflaterEngine.cs:402-420; 3 * HASH_SHIFT == HASH_BITS so older bytes fall out).
B200Z_HD uint32_t hash3(uint32_t b0, uint32_t b1, uint32_t b2) { return ((b0 << 10) ^ (b1 << 5) ^ b2) & 0x7FFFu; }

// Positions where the reference slides its window exactly when they are a loop top: there the first
// chain candidate at distance 32506 sits on window index 0 and is rejected by the zero sentinel (T8).
B200Z_HD bool is_slide_pos(uint32_t p) { return p >= kSlideFirst && ((p - kSlideFirst) & 32767u) == 0; }
// number of SlideWindow() calls performed once loop top `p` has been entered
B200Z_HD uint32_t slides_done(uint32_t p) { return p >= kSlideFirst ? ((p - kSlideFirst) >> 15) + 1 : 0; }

B200Z_HD uint32_t pack_match(uint32_t len, uint32_t dist) { return (len << 16) | dist; }
B200Z_HD uint32_t match_len(uint32_t m) { return m >> 16; }
B200Z_HD uint32_t match_dist(uint32_t m) { return m & 0xFFFFu; }

// ---- K2: one position's chain walk ------------------------------------------------------------
// data[q - bias], link[q - bias] address stream position q (bias lets a kernel pass shared-memory windows).
// Returns A = result with budget `chain`, B = result with budget `chain >> 2`, both from threshold 2 and with
// the nice-length early exit; 0 when no match of length >= 3 exists.
template <class DataT, class LinkT>
B200Z_HD void match_search(const DataT *data, const LinkT *link, uint32_t bias, uint32_t p, uint32_t n,
                           const LevelParams &lp, uint32_t &resA, uint32_t &resB, uint32_t abs_bias = 0) {
	resA = 0;
	resB = 0;
	const uint32_t la = n - p; // lookahead at a flushing loop top (or >= 262, where min() gives the same caps)
	if (la < (uint32_t)kMinMatch) return;
	uint32_t d = link[p - bias];
	if (d == 0) return;
	if (d > (uint32_t)kMaxDist - (is_slide_pos(p + abs_bias) ? 1u : 0u)) return; // DeflaterEngine.cs:788 + trap T8
	const uint32_t maxlen = la < (uint32_t)kMaxMatch ? la : (uint32_t)kMaxMatch;
	const uint32_t nice = la < (uint32_t)lp.nice ? la : (uint32_t)lp.nice;
	const DataT *s = data + (p - bias);
	uint32_t m = kMinMatch - 1, bd = 0;
	uint32_t dist = d;
	const uint32_t budgetB = (uint32_t)lp.chain >> 2;
	uint32_t cnt = 0;
	bool haveB = false;
	uint8_t scan_end1 = s[m - 1], scan_end = s[m];
	const uint8_t s0 = s[0], s1 = s[1];
	for (;;) {
		const DataT *c = s - dist;
		++cnt;
		if (c[m] == scan_end && c[m - 1] == scan_end1 && c[0] == s0 && c[1] == s1) {
			uint32_t l = 2;
			while (l < maxlen && c[l] == s[l]) ++l;
			if (l > m) {
				m = l;
				bd = dist;
				if (m >= nice) break;
				scan_end1 = s[m - 1];
				scan_end = s[m];
			}
		}
		if (cnt == budgetB) {
			resB = m >= (uint32_t)kMinMatch ? pack_match(m, bd) : 0;
			haveB = true;
		}
		if (cnt == (uint32_t)lp.chain) break;
		uint32_t l2 = link[(p - dist) - bias];
		if (l2 == 0) break;
		dist += l2;
		if (dist >= (uint32_t)kMaxDist) break; // chain entries need cur > limit, i.e. distance < 32506 (T7)
	}
	resA = m >= (uint32_t)kMinMatch ? pack_match(m, bd) : 0;
	if (!haveB) resB = resA;
}

// The rare case parse_step() cannot answer from the table: incoming threshold m0 >= nice (and < maxlen).
// Walks the first `budget` candidates for the first one strictly longer than m0 (which is then >= nice, so
// the reference stops there).  Returns packed match or 0.
template <class DataT, class LinkT>
B200Z_HDN uint32_t match_search_above(const DataT *data, const LinkT *link, uint32_t p, uint32_t n, uint32_t m0,
                                      uint32_t budget, uint32_t abs_bias = 0) {
	const uint32_t la = n - p;
	uint32_t d = link[p];
	if (d == 0 || d > (uint32_t)kMaxDist - (is_slide_pos(p + abs_bias) ? 1u : 0u)) return 0;
	const uint32_t maxlen = la < (uint32_t)kMaxMatch ? la : (uint32_t)kMaxMatch;
	uint32_t dist = d, cnt = 0;
	const DataT *s = data + p;
	for (;;) {
		const DataT *c = s - dist;
		++cnt;
		uint32_t l = 0;
		while (l < maxlen && c[l] == s[l]) ++l;
		if (l > m0) return pack_match(l, dist);
		if (cnt == budget) break;
		uint32_t l2 = link[p - dist];
		if (l2 == 0) break;
		dist += l2;
		if (dist >= (uint32_t)kMaxDist) break;
	}
	return 0;
}

// ---- K3: the lazy parse state machine (DeflaterEngine.DeflateSlow :741-855) --------------------
struct ParseState {
	uint32_t p;        // strstart as an input offset (window index = p + 1 - 32768 * slides)
	uint32_t mlen;     // matchLen
	uint32_t mstart;   // matchStart as an input offset
	uint32_t prevAvail; // prevAvailable
};

B200Z_HD void parse_init(ParseState &st) { // DeflaterEngine.Reset :234-253
	st.p = 0;
	st.mlen = kMinMatch - 1;
	st.mstart = 0;
	st.prevAvail = 0;
}

// symbol word: literal = byte value; match = (dist << 8) | (len - 3)
B200Z_HD uint32_t sym_lit(uint32_t b) { return b; }
B200Z_HD uint32_t sym_match(uint32_t len, uint32_t dist) { return (dist << 8) | (len - 3); }
B200Z_HD uint32_t sym_dist(uint32_t s) { return s >> 8; }
B200Z_HD uint32_t sym_len(uint32_t s) { return (s >> 8) ? (s & 0xFF) + 3 : 1; }

// One loop iteration of DeflateSlow at loop top st.p (< n).  `tab` holds (A, B) per position as uint2-like
// pairs; `emit(sym)` receives the tallied symbol (at most one per step).  strategy: 0 Default, 1 Filtered,
// 2 HuffmanOnly.  Returns the number of symbols emitted (0 or 1).
template <class TabFn, class DataFn, class SlowFn>
B200Z_HD int parse_step(ParseState &st, uint32_t n, const LevelParams &lp, int strategy, TabFn tab, DataFn byte_at,
                        SlowFn slow_search, uint32_t &out_sym) {
	const uint32_t p = st.p;
	const uint32_t prevLen = st.mlen, prevStart = st.mstart;
	const uint32_t la = n - p;
	if (la >= (uint32_t)kMinMatch && strategy != 2) {
		uint32_t a, b;
		tab(p, a, b);
		// (a | b) == 0 means either the head test failed (FindLongestMatch not entered) or no candidate of
		// length >= 3 exists.  Both leave (matchLen, matchStart) such that the decision below is the same:
		// the only side effect of an unproductive FindLongestMatch is the too-small/too-far discard of a
		// *carried* match, after which "matchLen <= prevLen" still holds and the previous match is emitted.
		if ((a | b) != 0) {
			// FindLongestMatch (:474-612)
			uint32_t m0 = st.mlen < (uint32_t)(kMinMatch - 1) ? (uint32_t)(kMinMatch - 1) : st.mlen;
			st.mlen = m0;
			const uint32_t maxlen = la < (uint32_t)kMaxMatch ? la : (uint32_t)kMaxMatch;
			bool ret;
			if (m0 >= maxlen) {
				ret = false; // "scan + matchLen > scanMax" (:488)
			} else {
				const uint32_t nice = la < (uint32_t)lp.nice ? la : (uint32_t)lp.nice;
				const bool quarter = m0 >= (uint32_t)lp.good;
				uint32_t r;
				if (m0 >= nice) r = slow_search(p, m0, quarter ? ((uint32_t)lp.chain >> 2) : (uint32_t)lp.chain);
				else r = quarter ? b : a;
				if (match_len(r) > m0) {
					st.mlen = match_len(r);
					st.mstart = p - match_dist(r);
				}
				ret = st.mlen >= (uint32_t)kMinMatch;
			}
			if (ret) {
				// discard match if too small and too far away (:794-797)
				if (st.mlen <= 5 && (strategy == 1 || (st.mlen == (uint32_t)kMinMatch && p - st.mstart > (uint32_t)kTooFar)))
					st.mlen = kMinMatch - 1;
			}
		}
	}
	int emitted = 0;
	if (prevLen >= (uint32_t)kMinMatch && st.mlen <= prevLen) {
		// previous match was better (:802-827)
		out_sym = sym_match(prevLen, p - 1 - prevStart);
		emitted = 1;
		st.p = p + prevLen - 1;
		st.prevAvail = 0;
		st.mlen = kMinMatch - 1;
	} else {
		if (st.prevAvail) {
			out_sym = sym_lit(byte_at(p - 1));
			emitted = 1;
		}
		st.prevAvail = 1;
		st.p = p + 1;
	}
	return emitted;
}

// A parse position with everything the next loop top depends on, plus the last loop top processed (needed for the
// window-slide count at block flush time, slides_done()).
struct ParseCarry {
	ParseState st;
	uint32_t last_top;
};
B200Z_HD bool carry_equal(const ParseCarry &a, const ParseCarry &b) {
	// matchStart is dead while matchLen < MIN_MATCH (it is only read for a pending match), so it must not keep two
	// otherwise identical states apart -- literal runs would never look converged
	const bool ms = (a.st.mlen < (uint32_t)kMinMatch && b.st.mlen < (uint32_t)kMinMatch) || a.st.mstart == b.st.mstart;
	return a.st.p == b.st.p && a.st.mlen == b.st.mlen && ms && a.st.prevAvail == b.st.prevAvail && a.last_top == b.last_top;
}

// Runs the loop tops in [c.st.p, seg_end) (clipped to n).  Returns the number of symbols tallied.  With EMIT, calls
// emit(k, sym, loop_top, bytes_after) for the k-th symbol of this run, bytes_after = input bytes covered by all
// symbols up to and including this one (what blockStart advances to when the block is cut here).
// The lazy parse is self-synchronising: started from a wrong state it normally falls in step with the true parse
// after a few symbols, which is what k_parse exploits (speculative segments + entry propagation until stable).
template <bool EMIT, class TabFn, class DataFn, class SlowFn, class EmitFn>
B200Z_HD uint32_t parse_run(ParseCarry &c, uint32_t seg_end, uint32_t n, const LevelParams &lp, int strategy, TabFn tab,
                            DataFn byte_at, SlowFn slow_search, EmitFn emit) {
	const uint32_t lim = seg_end < n ? seg_end : n;
	uint32_t cnt = 0;
	while (c.st.p < lim) {
		const uint32_t top = c.st.p;
		c.last_top = top;
		uint32_t sym = 0;
		if (parse_step(c.st, n, lp, strategy, tab, byte_at, slow_search, sym)) {
			if (EMIT) emit(cnt, sym, top, sym_dist(sym) ? top - 1 + sym_len(sym) : top);
			++cnt;
		}
	}
	return cnt;
}

// ---- levels 1-4: DeflaterEngine.DeflateFast (:651-739) -----------------------------------------------
// In the greedy levels the hash chains depend on the parse (positions inside a match longer than max_lazy are not
// inserted, :699-715), so a stream is parsed serially, with the reference's own data structures: head[]/prev[] hold
// 16-bit WINDOW indices, SlideWindow (:441-462) re-bases them, and the zero sentinel, the FillWindow schedule (:366-400)
// and the "strstart > 65274" slide test (:668) are reproduced literally.  The 64 KiB window itself is not copied:
// window[w] is input byte  w - 1 + 32768 * slides.  One thread per stream; all streams of a batch run concurrently.
//
// Call pattern emulated: SetInput(all) -> Deflate() until IsNeedingInput (DeflaterOutputStream.Write :506-510) -> Finish()
// (or Flush()) -> drain.  emit(sym) receives the tallied symbols; block(byte_start, stored_ok) is called for every
// FlushBlock with the block's first input byte and whether storedOffset >= 0 (trap T4).
struct FastEngine {
	uint32_t n;           // stream bytes handed over so far (inputEnd, counted from the start of the stream)
	const uint8_t *in;    // the slot: history (a dictionary, or the last bytes of earlier segments) followed by the data
	uint32_t slot_len;    // bytes in the slot
	uint32_t woff;        // window index w holds slot byte w + woff (= 32768 * slides - 1 - stream offset of slot byte 0)
	uint16_t *head;       // 32768 entries, zeroed by the caller
	uint16_t *prev;       // 32768 entries, zeroed by the caller
	int strstart, blockStart, lookahead, matchStart, matchLen, ins_h;
	uint32_t slides;      // number of SlideWindow calls so far
	uint32_t inputOff;    // stream bytes handed to the window so far
	uint32_t nsym;        // symbols tallied in the current block
	int coop;             // 1: never slide inside the engine, report kFeNeedSlide instead (the kernel slides warp-wide)
	                      // 2: also report kFeGroup at a loop top from which the kernel's warp-wide group step may run
};
constexpr int kFeFalse = 0, kFeTrue = 1, kFeNeedSlide = 2, kFeGroup = 3;
constexpr int kFeGroupMin = 8; // fewer steady-state loop tops than this ahead: the serial loop takes them

// How many of the next DeflateFast loop tops (strstart, strstart + 1, ...) are certain to be steady-state iterations
// whatever the parse does: lookahead >= MIN_LOOKAHEAD at each (so maxlen = 258, niceLength = nice, every lookahead test of
// :684-:715 true), no SlideWindow due (:668), no full block (:718) -- a literal or a match per loop top at most.
B200Z_HD int fe_group_lanes(int strstart, int lookahead, uint32_t nsym) {
	int nl = 32;
	const int a = lookahead - (kMaxMatch + kMinMatch + 1) + 1;
	const int b = 2 * kWSize - (kMaxMatch + kMinMatch + 1) + 1 - strstart;
	const int c = kBlockSyms - 1 - (int)nsym;
	if (a < nl) nl = a;
	if (b < nl) nl = b;
	if (c < nl) nl = c;
	return nl;
}

// What DeflateFast carries from one Deflate() call to the next besides head[] / prev[] (DeflaterEngine's fields): saved
// when a segment ends with Flush(), loaded when the stream goes on (b200z_history.engine_state).
struct FastCarry {
	int32_t strstart, blockStart, lookahead, matchStart, matchLen, ins_h;
	uint32_t slides, inputOff;
};
constexpr int kFastStateBytes = 2 * 65536 + 64; // head[32768], prev[32768], FastCarry

// inputOff and 32768 * slides only matter relative to each other and to the window (strstart and blockStart are window
// indices, the phase of SlideWindow): a run entered with carried state drops the same multiple of 32768 from both, so that
// no 32-bit field holds a stream-absolute position and a stream may go on past 4 GiB.  Returns the multiple dropped.
B200Z_HD uint32_t carry_rebase(uint32_t &slides, uint32_t &inputOff) {
	const uint32_t m = slides > 1u ? slides - 1u : 0u;
	slides -= m;
	inputOff -= 32768u * m;
	return m;
}
// stream position (dictionary included, reduced like inputOff) of window index w
B200Z_HD uint32_t fe_stream_pos(uint32_t slides, int w) { return 32768u * slides - 1u + (uint32_t)w; }

B200Z_HD uint32_t fe_win(const FastEngine &e, int w) { return (uint32_t)e.in[(uint32_t)w + e.woff]; }

B200Z_HD void fe_init(FastEngine &e, const uint8_t *in, uint32_t n, uint16_t *head, uint16_t *prev) {
	e.n = n;
	e.in = in;
	e.slot_len = n;
	e.woff = 0xFFFFFFFFu; // window index 1 is slot byte 0 (DeflaterEngine.cs:91-93)
	e.head = head;
	e.prev = prev;
	e.strstart = e.blockStart = 1; // DeflaterEngine.cs:91-93
	e.lookahead = 0;
	e.matchStart = 0;
	e.matchLen = kMinMatch - 1;
	e.ins_h = 0;
	e.slides = 0;
	e.inputOff = 0;
	e.nsym = 0;
	e.coop = 0;
}
B200Z_HD void fe_save(const FastEngine &e, FastCarry &c) {
	c.strstart = e.strstart;
	c.blockStart = e.blockStart;
	c.lookahead = e.lookahead;
	c.matchStart = e.matchStart;
	c.matchLen = e.matchLen;
	c.ins_h = e.ins_h;
	c.slides = e.slides;
	c.inputOff = e.inputOff;
}
// the stream goes on: the slot holds its last `hist` bytes followed by the new data (the tables are the caller's business)
B200Z_HD void fe_load(FastEngine &e, const FastCarry &c, const uint8_t *slot, uint32_t slot_len, uint32_t hist, uint16_t *head,
                      uint16_t *prev) {
	e.in = slot;
	e.slot_len = slot_len;
	e.head = head;
	e.prev = prev;
	e.strstart = c.strstart;
	e.blockStart = c.blockStart;
	e.lookahead = c.lookahead;
	e.matchStart = c.matchStart;
	e.matchLen = c.matchLen;
	e.ins_h = c.ins_h;
	e.slides = c.slides;
	e.inputOff = c.inputOff;
	carry_rebase(e.slides, e.inputOff);
	e.n = e.inputOff; // nothing new is visible before the first SetInput of the segment
	// slot byte `hist` is window index blockStart: the first byte no block has taken yet (behind a Flush() also strstart;
	// behind the cut of an open run the bytes from there to inputOff are already in the window as lookahead)
	e.woff = (uint32_t)hist - (uint32_t)c.blockStart;
	e.nsym = 0;
	e.coop = 0;
}

B200Z_HD void fe_update_hash(FastEngine &e) { e.ins_h = (int)((fe_win(e, e.strstart) << 5) ^ fe_win(e, e.strstart + 1)); } // :402-410

B200Z_HD int fe_insert_string(FastEngine &e) { // :417-439
	const int hash = (int)(((uint32_t)e.ins_h << 5) ^ fe_win(e, e.strstart + 2)) & 0x7FFF;
	const uint16_t match = e.head[hash];
	e.prev[e.strstart & 32767] = match;
	e.head[hash] = (uint16_t)e.strstart;
	e.ins_h = hash;
	return (int)match;
}

// DeflaterEngine.SetDictionary (:198-229): the dictionary (>= MIN_MATCH bytes, already cut to its last MAX_DIST bytes)
// sits in front of the data in the same buffer; every position but its last two is inserted
B200Z_HDN void fe_set_dictionary(FastEngine &e, uint32_t dict_len) {
	if (dict_len < (uint32_t)kMinMatch) return;
	fe_update_hash(e);
	for (uint32_t k = 0; k + 2 < dict_len; ++k) {
		fe_insert_string(e);
		++e.strstart;
	}
	e.strstart += 2;
	e.blockStart = e.strstart;
	e.inputOff = dict_len;
}

B200Z_HD void fe_slide_scalars(FastEngine &e) { // :443-446
	e.matchStart -= kWSize;
	e.strstart -= kWSize;
	e.blockStart -= kWSize;
	e.slides += 1;
	e.woff += (uint32_t)kWSize;
}
B200Z_HDN void fe_slide(FastEngine &e) { // :441-462
	fe_slide_scalars(e);
	for (int i = 0; i < 32768; ++i) {
		const int m = e.head[i];
		e.head[i] = (uint16_t)(m >= kWSize ? m - kWSize : 0);
	}
	for (int i = 0; i < 32768; ++i) {
		const int m = e.prev[i];
		e.prev[i] = (uint16_t)(m >= kWSize ? m - kWSize : 0);
	}
}

// returns false (and does nothing) when a slide is due and the engine runs in cooperative mode
B200Z_HD bool fe_fill_window(FastEngine &e) { // :366-400
	if (e.strstart >= kWSize + kMaxDist) {
		if (e.coop) return false;
		fe_slide(e);
	}
	if (e.lookahead < kMaxMatch + kMinMatch + 1 && e.inputOff < e.n) {
		uint32_t more = (uint32_t)(2 * kWSize - e.lookahead - e.strstart);
		if (more > e.n - e.inputOff) more = e.n - e.inputOff;
		e.inputOff += more;
		e.lookahead += (int)more;
	}
	if (e.lookahead >= kMinMatch) fe_update_hash(e);
	return true;
}

// four window bytes starting at window index w, first byte in the low bits.  The device reads two aligned words (the input
// slot is 256-byte aligned and has 16 bytes of slack behind n); the host copy stays inside [0, n).
B200Z_HD uint32_t fe_word(const FastEngine &e, int w) {
	const uint32_t a = (uint32_t)w + e.woff;
#ifdef __CUDA_ARCH__
	const uint32_t *p = reinterpret_cast<const uint32_t *>(e.in + (a & ~3u));
	return __funnelshift_r(p[0], p[1], (a & 3u) * 8u);
#else
	uint32_t v = 0;
	for (uint32_t k = 0; k < 4 && a + k < e.slot_len; k++) v |= (uint32_t)e.in[a + k] << (8 * k);
	return v;
#endif
}
B200Z_HD uint32_t fe_ctz(uint32_t x) {
#ifdef __CUDA_ARCH__
	return (uint32_t)(__ffs((int)x) - 1);
#else
	return (uint32_t)__builtin_ctz(x);
#endif
}

B200Z_HDN bool fe_find_longest_match(FastEngine &e, int curMatch, const LevelParams &lp) { // :474-612
	const int scan0 = e.strstart;
	const int maxlen = e.lookahead < kMaxMatch ? e.lookahead : kMaxMatch;
	const int scanMax = scan0 + maxlen - 1;
	const int limit = scan0 - kMaxDist > 0 ? scan0 - kMaxDist : 0;
	int chainLength = lp.chain;
	const int niceLength = lp.nice < e.lookahead ? lp.nice : e.lookahead;
	if (e.matchLen < kMinMatch - 1) e.matchLen = kMinMatch - 1;
	if (scan0 + e.matchLen > scanMax) return false;
	uint32_t scan_end1 = fe_win(e, scan0 + e.matchLen - 1), scan_end = fe_win(e, scan0 + e.matchLen);
	const uint32_t s0 = fe_win(e, scan0), s1 = fe_win(e, scan0 + 1);
	if (e.matchLen >= lp.good) chainLength >>= 2;
	do {
		const int match = curMatch;
		if (fe_win(e, match + e.matchLen) == scan_end && fe_win(e, match + e.matchLen - 1) == scan_end1 &&
		    fe_win(e, match) == s0 && fe_win(e, match + 1) == s1) {
			// the reference extends byte by byte (:548-590); four bytes per compare give the same length
			int l = 2;
			while (l + 4 <= maxlen) {
				const uint32_t x = fe_word(e, match + l) ^ fe_word(e, scan0 + l);
				if (x) {
					l += (int)(fe_ctz(x) >> 3);
					goto extended;
				}
				l += 4;
			}
			while (l < maxlen && fe_win(e, match + l) == fe_win(e, scan0 + l)) ++l;
		extended:
			if (l > e.matchLen) {
				e.matchStart = curMatch;
				e.matchLen = l;
				if (e.matchLen >= niceLength) break;
				scan_end1 = fe_win(e, scan0 + l - 1);
				scan_end = fe_win(e, scan0 + l);
			}
		}
	} while ((curMatch = (int)e.prev[curMatch & 32767]) > limit && 0 != --chainLength);
	return e.matchLen >= kMinMatch;
}

// DeflateFast (:651-739).  Returns the reference's `progress` value (kFeFalse / kFeTrue), or kFeNeedSlide in cooperative
// mode: nothing has been done at the current loop top then, and calling again after the slide resumes transparently.
template <class EmitFn, class BlockFn>
B200Z_HDN int fe_deflate_fast(FastEngine &e, bool flush, bool finish, const LevelParams &lp, int strategy, EmitFn emit,
                               BlockFn block) {
	const int kMinLookahead = kMaxMatch + kMinMatch + 1;
	if (e.lookahead < kMinLookahead && !flush) return kFeFalse;
	while (e.lookahead >= kMinLookahead || flush) {
		if (e.lookahead == 0) {
			// we are flushing everything
			block((uint32_t)e.blockStart + e.woff, e.blockStart >= 0, finish);
			e.nsym = 0;
			e.blockStart = e.strstart;
			return kFeFalse;
		}
		if (e.strstart > 2 * kWSize - kMinLookahead) {
			if (e.coop) return kFeNeedSlide;
			fe_slide(e);
		}
		if (e.coop == 2 && strategy != 2 && fe_group_lanes(e.strstart, e.lookahead, e.nsym) >= kFeGroupMin) return kFeGroup;
		int hashHead;
		if (e.lookahead >= kMinMatch && (hashHead = fe_insert_string(e)) != 0 && strategy != 2 &&
		    e.strstart - hashHead <= kMaxDist && fe_find_longest_match(e, hashHead, lp)) {
			emit(sym_match((uint32_t)e.matchLen, (uint32_t)(e.strstart - e.matchStart)));
			const bool full = ++e.nsym >= (uint32_t)kBlockSyms;
			e.lookahead -= e.matchLen;
			if (e.matchLen <= lp.lazy && e.lookahead >= kMinMatch) {
				while (--e.matchLen > 0) {
					++e.strstart;
					fe_insert_string(e);
				}
				++e.strstart;
			} else {
				e.strstart += e.matchLen;
				if (e.lookahead >= kMinMatch - 1) fe_update_hash(e);
			}
			e.matchLen = kMinMatch - 1;
			if (!full) continue;
		} else {
			// no match found
			emit(sym_lit(fe_win(e, e.strstart)));
			++e.nsym;
			++e.strstart;
			--e.lookahead;
		}
		if (e.nsym >= (uint32_t)kBlockSyms) {
			const bool lastBlock = finish && e.lookahead == 0;
			block((uint32_t)e.blockStart + e.woff, e.blockStart >= 0, lastBlock);
			e.nsym = 0;
			e.blockStart = e.strstart;
			return lastBlock ? kFeFalse : kFeTrue;
		}
	}
	return kFeTrue;
}

// One segment of a stream (everything up to a Flush() or Finish()), call pattern above.  The segment's bytes arrive in
// `nchunks` SetInput calls, cum[i] bytes after the first i + 1 of them (nchunks == 0: one call with everything); each is
// followed by Deflate() until IsNeedingInput.  For DeflateFast the result depends on that schedule (trap T9: FillWindow
// slides at strstart >= 65274 when it is called, DeflateFast at > 65274), so the handle records it.  The segment's data
// starts at blockStart (the first byte no block has taken; after a cut some of it may already sit in the window).
// end_mode: B200Z_END_* (0 finish, 1 flush then finish, 2 flush, 3 none).
// End mode 3 is an open run: only the BUSY_STATE loops run, over every call of the schedule (busy_last is ignored), and
// blocks end only by the 16384-symbol rule.  Right behind every block that closes, DeflateFast returns and the engine
// carries nothing but its window, tables and scalars (strstart == blockStart, no symbol pending): cut(ci) is called there
// with the index of the call in whose Deflate() loop the block closed.  The last cut is where the next run starts: its
// schedule is the rest of call ci, from blockStart on, followed by the later calls.
template <class EmitFn, class BlockFn, class CutFn>
B200Z_HDN void fe_run(FastEngine &e, const LevelParams &lp, int strategy, int end_mode, EmitFn emit, BlockFn block, CutFn cut,
                      const uint32_t *cum, int nchunks, bool busy_last) {
	const bool open = end_mode == 3;
	const uint32_t seg_base = fe_stream_pos(e.slides, e.blockStart);
	const uint32_t seg_end = 32768u * e.slides - 1u - e.woff + e.slot_len; // stream position behind the slot
	// busy_last = false: Flush() / Finish() follows the last SetInput directly, without a Deflate() call in between
	const int nc = nchunks > 0 ? nchunks : 1;
	bool closed = false;
	auto blk = [&](uint32_t start, bool ok, bool last) {
		block(start, ok, last);
		closed = true;
	};
	for (int ci = 0; ci < nc; ci++) {
		e.n = nchunks > 0 ? seg_base + cum[ci] : seg_end;
		if (ci == nc - 1 && !busy_last && !open) break;
		// BUSY_STATE: Deflater.Deflate -> engine.Deflate(false, false) until it reports "needs input" (:104-137)
		for (;;) {
			fe_fill_window(e);
			closed = false;
			const int r = fe_deflate_fast(e, false, false, lp, strategy, emit, blk);
			if (open && closed) cut(ci);
			if (r == kFeFalse) break;
		}
	}
	if (open) return;
	// Flush() or Finish(): engine.Deflate(flush, finish) runs the function with canFlush = flush && inputOff == inputEnd
	// (DeflaterEngine.cs:104-137) -- false as long as part of an undrained last SetInput is still outside the window
	const bool finish = end_mode == 0;
	for (;;) {
		fe_fill_window(e);
		if (fe_deflate_fast(e, e.inputOff == e.n, finish, lp, strategy, emit, blk) == kFeFalse) break;
	}
	// (end_mode 1: the sync padding and the final empty static block that Finish() adds are appended by k_scan)
}
template <class EmitFn, class BlockFn>
B200Z_HDN void fe_run(FastEngine &e, const LevelParams &lp, int strategy, int end_mode, EmitFn emit, BlockFn block,
                      const uint32_t *cum = nullptr, int nchunks = 0, bool busy_last = true) {
	fe_run(e, lp, strategy, end_mode, emit, block, [](int) {}, cum, nchunks, busy_last);
}

// ---- level 0: DeflaterEngine.DeflateStored (:614-649) --------------------------------------------------
// Only block boundaries are decided here (pure integer bookkeeping); block(byte_start, length, last) is called for
// every FlushStoredBlock.  Same call pattern as fe_run.  Sync-flush padding is skipped at level 0 (Deflater.cs:488).
// What DeflateStored carries from one Deflate() call to the next (b200z_history.stored_state, in/out).
struct StoredCarry {
	int32_t strstart, blockStart;
	uint32_t slides, inputOff;
};
// A stream going on from a carried state (a flush, or the cut of an open run): the state rebased (carry_rebase), and the
// start_bias for stored_run when the data sits behind `hist` bytes of history in the slot -- the data starts at blockStart.
B200Z_HD uint32_t stored_rebase(StoredCarry &c, uint32_t hist) {
	carry_rebase(c.slides, c.inputOff);
	return (uint32_t)(c.blockStart - 1) + 32768u * c.slides - hist;
}
// One segment of n bytes in `nchunks` SetInput calls (cum[] as for fe_run; stored-block boundaries depend on the schedule,
// trap T9).  `carry`: in = the state a flushed earlier segment or the cut of an open run left (NULL: start of the stream,
// dict_len bytes of preset dictionary in front); out = the state after this segment.  Block starts are stream offsets minus
// `start_bias` (the stream offset of the first byte block starts are counted from, in the frame of carry_in's slides).
// end_mode 3 (open run, as for fe_run): the BUSY_STATE loops only, over every call; `carry_out` is the state right behind
// the last block that closed (the entry state if none did), *cut_call the call in whose Deflate() loop that happened.
// Behind such a cut strstart may lie ahead of blockStart (a block ends at MAX_BLOCK_SIZE): those bytes are in the window.
template <class BlockFn>
inline void stored_run(uint32_t n, uint32_t dict_len, int end_mode, BlockFn block, const uint32_t *cum = nullptr, int nchunks = 0,
                       const StoredCarry *carry_in = nullptr, StoredCarry *carry_out = nullptr, uint32_t start_bias = 0,
                       bool busy_last = true, int *cut_call = nullptr) {
	// host only: run when a plan is built
	// dict_len: a preset dictionary in front of the n data bytes (SetDictionary leaves strstart = blockStart = 1 + length)
	int strstart = 1 + (int)dict_len, blockStart = 1 + (int)dict_len, lookahead = 0;
	uint32_t slides = 0, inputOff = 0;
	if (carry_in) {
		strstart = carry_in->strstart;
		blockStart = carry_in->blockStart;
		slides = carry_in->slides;
		inputOff = carry_in->inputOff;
	}
	const bool open = end_mode == 3;
	// the data starts at blockStart; inputOff (lookahead is 0 between calls) is strstart - blockStart bytes further on
	const uint32_t seg_base = inputOff - (uint32_t)(strstart - blockStart);
	uint32_t vis = seg_base; // inputEnd: stream bytes handed over so far
	const int kMaxBlock = 65531; // DeflaterConstants.MAX_BLOCK_SIZE
	auto fill = [&]() {
		if (strstart >= kWSize + kMaxDist) {
			strstart -= kWSize;
			blockStart -= kWSize;
			slides += 1;
		}
		if (lookahead < kMaxMatch + kMinMatch + 1 && inputOff < vis) {
			uint32_t more = (uint32_t)(2 * kWSize - lookahead - strstart);
			if (more > vis - inputOff) more = vis - inputOff;
			inputOff += more;
			lookahead += (int)more;
		}
	};
	bool closed = false;
	auto stored = [&](bool flush, bool finish) -> bool {
		if (!flush && lookahead == 0) return false;
		strstart += lookahead;
		lookahead = 0;
		int storedLength = strstart - blockStart;
		if (storedLength >= kMaxBlock || (blockStart < kWSize && storedLength >= kMaxDist) || flush) {
			bool lastBlock = finish;
			if (storedLength > kMaxBlock) {
				storedLength = kMaxBlock;
				lastBlock = false;
			}
			// window index w is stream byte w - 1 + 32768 * slides minus what the dictionary took (it is not stream data)
			block((uint32_t)(blockStart - 1) + 32768u * slides - start_bias, (uint32_t)storedLength, lastBlock);
			blockStart += storedLength;
			closed = true;
			return !(lastBlock || storedLength == 0);
		}
		return true;
	};
	auto save = [&](StoredCarry *c) {
		if (!c) return;
		c->strstart = strstart;
		c->blockStart = blockStart;
		c->slides = slides;
		c->inputOff = inputOff;
	};
	save(carry_out);
	if (cut_call) *cut_call = 0;
	const int nc = nchunks > 0 ? nchunks : 1;
	for (int ci = 0; ci < nc; ci++) {
		vis = seg_base + (nchunks > 0 ? cum[ci] : n);
		if (ci == nc - 1 && !busy_last && !open) break;
		for (;;) {
			fill();
			closed = false;
			const bool more = stored(false, false);
			if (open && closed) {
				save(carry_out);
				if (cut_call) *cut_call = ci;
			}
			if (!more) break;
		}
	}
	if (open) return;
	const bool finish = end_mode == 0;
	for (;;) {
		fill();
		if (!stored(inputOff == vis, finish)) break;
	}
	if (end_mode == 1) {
		for (;;) {
			fill();
			if (!stored(inputOff == vis, true)) break;
		}
	}
	save(carry_out);
}

// ---- DeflaterHuffman.cs helpers ----------------------------------------------------------------
// floor(log2(x)) for x > 0
B200Z_HD int ilog2(uint32_t x) {
#ifdef __CUDA_ARCH__
	return 31 - __clz((int)x);
#else
	return 31 - __builtin_clz(x);
#endif
}
// Lcode :932-946 (argument is length - 3).  The reference halves len_m3 until it is below 8, adding 4 per halving: that is
// ilog2(len_m3) - 2 halvings, in closed form so that the lanes of a warp do not diverge on the loop.
B200Z_HD int lcode(int len_m3) {
	if (len_m3 == 255) return 285;
	if (len_m3 < 8) return 257 + len_m3;
	const int k = ilog2((uint32_t)len_m3) - 2;
	return 257 + 4 * k + (len_m3 >> k);
}
// Dcode :948-957 (argument is distance - 1): ilog2(dist_m1) - 1 halvings of 2 each, likewise
B200Z_HD int dcode(int dist_m1) {
	if (dist_m1 < 4) return dist_m1;
	const int k = ilog2((uint32_t)dist_m1) - 1;
	return 2 * k + (dist_m1 >> k);
}
B200Z_HD int lcode_extra_bits(int lc) { // CompressBlock :716-720
	int bits = (lc - 261) / 4;
	return (bits > 0 && bits <= 5) ? bits : 0;
}
B200Z_HD int dcode_extra_bits(int dc) { // CompressBlock :725-729
	int bits = dc / 2 - 1;
	return bits > 0 ? bits : 0;
}
B200Z_HD uint32_t bit_reverse16(uint32_t v) { // BitReverse :924-930
	v = ((v & 0x5555u) << 1) | ((v >> 1) & 0x5555u);
	v = ((v & 0x3333u) << 2) | ((v >> 2) & 0x3333u);
	v = ((v & 0x0F0Fu) << 4) | ((v >> 4) & 0x0F0Fu);
	v = ((v & 0x00FFu) << 8) | ((v >> 8) & 0x00FFu);
	return v & 0xFFFFu;
}
B200Z_HD int static_llen(int i) { return i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8)); } // :611-630
B200Z_HD uint32_t static_lcode(int i) {
	if (i < 144) return bit_reverse16((uint32_t)(0x030 + i) << 8);
	if (i < 256) return bit_reverse16((uint32_t)(0x190 - 144 + i) << 7);
	if (i < 280) return bit_reverse16((uint32_t)(0x000 - 256 + i) << 9);
	return bit_reverse16((uint32_t)(0x0c0 - 280 + i) << 8);
}
B200Z_HD uint32_t static_dcode(int i) { return bit_reverse16((uint32_t)i << 11); } // :637-641, length 5

// Tree.BuildTree + BuildLength (DeflaterHuffman.cs:196-329, :475-579), operation for operation.
//   freqs[numSymbols] in; length[numSymbols], bl_counts[maxLength], numCodes out.
//   scratch (tree_scratch_ints(numSymbols) ints, 8-byte aligned): heap[numSymbols + 1] entries of (value, node), then childs[4*L-2]
//   as 16-bit node numbers (< 2 * L - 1, or -1), then lengths[2*L-1] bytes (<= maxLength), with L <= numSymbols leaves.  The
//   reference's values[] array is only ever written (the heap reads its copy), so it is not kept.
// Each heap entry holds its node's value next to the node number, so that a heap step reads and writes one 8-byte entry
// per child: the tree is built by a single thread, its time is the sum of these load latencies, and with many CTAs on an
// SM the shared-memory instructions of all their tree builds share one pipe.
struct alignas(8) HeapEnt {
	int32_t val, node;
};
B200Z_HDN int build_tree(const int *freqs, int numSymbols, int minNumCodes, int maxLength, uint8_t *length,
                         int *bl_counts, int *scratch) {
	HeapEnt *heap = reinterpret_cast<HeapEnt *>(scratch);
	int heapLen = 0;
	int maxCode = 0;
	for (int n = 0; n < numSymbols; n++) {
		int freq = freqs[n];
		if (freq != 0) {
			int pos = heapLen++;
			int ppos;
			while (pos > 0 && freqs[heap[ppos = (pos - 1) / 2].node] > freq) {
				heap[pos].node = heap[ppos].node;
				pos = ppos;
			}
			heap[pos].node = n;
			maxCode = n;
		}
	}
	while (heapLen < 2) {
		int node = maxCode < 2 ? ++maxCode : 0;
		heap[heapLen++].node = node;
	}
	int numCodes = (maxCode + 1 > minNumCodes) ? maxCode + 1 : minNumCodes;
	int numLeafs = heapLen;
	int16_t *childs = reinterpret_cast<int16_t *>(heap + numSymbols + 1);       // 4*heapLen - 2
	uint8_t *lengths = reinterpret_cast<uint8_t *>(childs + (4 * numLeafs - 2)); // 2*heapLen - 1
	int numNodes = numLeafs;
	for (int i = 0; i < heapLen; i++) {
		int node = heap[i].node;
		childs[2 * i] = (int16_t)node;
		childs[2 * i + 1] = -1;
		heap[i] = HeapEnt{freqs[node] << 8, i};
	}
	// heap[heapLen] is kept above every value: a node whose right child would be heap[heapLen] then takes its left child, as
	// the reference's "path + 1 < heapLen" test decides, without the test
	heap[heapLen] = HeapEnt{0x7FFFFFFF, -1};
	do {
		const HeapEnt top = heap[0];
		const int first = top.node, firstVal = top.val;
		const HeapEnt bottom = heap[--heapLen];
		heap[heapLen].val = 0x7FFFFFFF;
		int last = bottom.node;
		int lastVal = bottom.val;
		int ppos = 0;
		int path = 1;
		while (path < heapLen) {
			// both children are fetched before the comparison decides
			const HeapEnt e0 = heap[path], e1 = heap[path + 1];
			const bool right = e0.val > e1.val;
			if (right) path++;
			heap[ppos] = right ? e1 : e0;
			ppos = path;
			path = path * 2 + 1;
		}
		while ((path = ppos) > 0 && heap[ppos = (path - 1) / 2].val > lastVal) heap[path] = heap[ppos];
		heap[path] = HeapEnt{lastVal, last};
		const HeapEnt sec = heap[0];
		const int second = sec.node, secondVal = sec.val;
		last = numNodes++;
		childs[2 * last] = (int16_t)first;
		childs[2 * last + 1] = (int16_t)second;
		int d1 = firstVal & 0xff, d2 = secondVal & 0xff;
		int mindepth = d1 < d2 ? d1 : d2;
		lastVal = firstVal + secondVal - mindepth + 1;
		ppos = 0;
		path = 1;
		while (path < heapLen) {
			const HeapEnt e0 = heap[path], e1 = heap[path + 1];
			const bool right = e0.val > e1.val;
			if (right) path++;
			heap[ppos] = right ? e1 : e0;
			ppos = path;
			path = ppos * 2 + 1;
		}
		while ((path = ppos) > 0 && heap[ppos = (path - 1) / 2].val > lastVal) heap[path] = heap[ppos];
		heap[path] = HeapEnt{lastVal, last};
	} while (heapLen > 1);

	// BuildLength (:475-579); childs.Length / 2 == numNodes == 2 * numLeafs - 1
	for (int i = 0; i < numSymbols; i++) length[i] = 0;
	int overflow = 0;
	for (int i = 0; i < maxLength; i++) bl_counts[i] = 0;
	lengths[numNodes - 1] = 0;
	for (int i = numNodes - 1; i >= 0; i--) {
		if (childs[2 * i + 1] != -1) {
			int bitLength = lengths[i] + 1;
			if (bitLength > maxLength) {
				bitLength = maxLength;
				overflow++;
			}
			lengths[childs[2 * i]] = lengths[childs[2 * i + 1]] = (uint8_t)bitLength;
		} else {
			int bitLength = lengths[i];
			bl_counts[bitLength - 1]++;
			length[childs[2 * i]] = (uint8_t)lengths[i];
		}
	}
	if (overflow == 0) return numCodes;
	int incrBitLen = maxLength - 1;
	do {
		while (bl_counts[--incrBitLen] == 0) {
		}
		do {
			bl_counts[incrBitLen]--;
			bl_counts[++incrBitLen]++;
			overflow -= 1 << (maxLength - 1 - incrBitLen);
		} while (overflow > 0 && incrBitLen < maxLength - 1);
	} while (overflow > 0);
	bl_counts[maxLength - 1] += overflow;
	bl_counts[maxLength - 2] -= overflow;
	int nodePtr = 2 * numLeafs;
	for (int bits = maxLength; bits != 0; bits--) {
		int n = bl_counts[bits - 1];
		while (n > 0) {
			int childPtr = 2 * childs[nodePtr++];
			if (childs[childPtr + 1] == -1) {
				length[childs[childPtr]] = (uint8_t)bits;
				n--;
			}
		}
	}
	return numCodes;
}

// Tree.BuildCodes (:151-194): canonical codes, left-aligned in 16 bits then bit-reversed.
B200Z_HDN void build_codes(const uint8_t *length, const int *bl_counts, int maxLength, int numCodes, uint16_t *codes) {
	int nextCode[15];
	int code = 0;
	for (int bits = 0; bits < maxLength; bits++) {
		nextCode[bits] = code;
		code += bl_counts[bits] << (15 - bits);
	}
	for (int i = 0; i < numCodes; i++) {
		int bits = length[i];
		if (bits > 0) {
			codes[i] = (uint16_t)bit_reverse16((uint32_t)nextCode[bits - 1]);
			nextCode[bits - 1] += 1 << (16 - bits);
		} else {
			codes[i] = 0;
		}
	}
}

// LSB-first bit writer over 32-bit words owned by ONE thread (block headers).  The destination words must be
// zero; the content is what PendingBuffer.WriteBits (:168-189) would have produced for the same calls.
struct BitSink {
	uint32_t *w;
	uint32_t nbits;
	B200Z_HD void put(uint32_t v, int count) {
		if (count == 0) return;
		uint32_t idx = nbits >> 5, sh = nbits & 31;
		w[idx] |= v << sh;
		if (sh + count > 32) w[idx + 1] |= v >> (32 - sh);
		nbits += count;
	}
};
struct BitCounter {
	uint32_t nbits;
	B200Z_HD void put(uint32_t, int count) { nbits += count; }
};

// Tree.CalcBLFreq (:349-405) and Tree.WriteTree (:411-473) share one run-length walk; Sink decides what a
// visit does.  visit(symbol) for a bit-length symbol, extra(value, bits) for the repeat counts.
// The walk's steps never cross from one run of equal code lengths into the next (its inner loop stops at the first
// different length, and the first step of a run of a nonzero length always sees curlen != nextlen), so what a run emits
// depends on its length value and its size alone: walk_code_run() is that, and k_plan runs it for all runs at once.
template <class Visit, class Extra>
B200Z_HD void walk_code_run(int len, int run, Visit visit, Extra extra) {
	const int max_count = len == 0 ? 138 : 6;
	if (len != 0) {
		visit(len);
		run--;
	}
	while (run > 0) {
		const int count = run < max_count ? run : max_count;
		run -= count;
		if (count < 3) {
			for (int k = 0; k < count; k++) visit(len);
		} else if (len != 0) {
			visit(16);
			extra(count - 3, 2);
		} else if (count <= 10) {
			visit(17);
			extra(count - 3, 3);
		} else {
			visit(18);
			extra(count - 11, 7);
		}
	}
}
template <class Visit, class Extra>
B200Z_HD void walk_code_lengths(const uint8_t *length, int numCodes, Visit visit, Extra extra) {
	int i = 0;
	while (i < numCodes) {
		int j = i + 1;
		while (j < numCodes && length[j] == length[i]) j++;
		walk_code_run(length[i], j - i, visit, extra);
		i = j;
	}
}

// BL_ORDER (DeflaterHuffman.cs:33): the order in which the bit-length code lengths are sent
B200Z_HD int bl_order(int i) {
	if (i < 3) return 16 + i;
	if (i == 3) return 0;
	return (i & 1) ? 7 - ((i - 5) >> 1) : 8 + ((i - 4) >> 1);
}
// FlushBlock's choice (:830-857) from opt_len (dynamic trees, header included) and static_len: 0 stored, 1 static, 2 dynamic
B200Z_HD int block_type(int stored_ok, int storedLength, int opt_len, int static_len) {
	if (opt_len >= static_len) opt_len = static_len; // force static trees
	if (stored_ok && storedLength + 4 < (opt_len >> 3)) return 0;
	return opt_len == static_len ? 1 : 2;
}

// Everything FlushBlock (:788-857) decides for one block, from its histograms.
struct BlockPlan {
	int type;           // 0 stored, 1 static, 2 dynamic
	int lit_numCodes, dist_numCodes, blTreeCodes;
	int opt_len, static_len;
	uint32_t hdr_bits;  // 3 header bits (+ tree description for dynamic blocks); stored: 3
	uint32_t body_bits; // symbols + EOB (stored: 0; the payload is byte-aligned separately)
};

// freqs are the literal (286) and distance (30) histograms with EOB already counted; extra_bits as tallied by
// TallyDist (:894-916).  Outputs code lengths / codes for the block's chosen trees and, for dynamic blocks, the
// header bit string into hdr_words (zeroed by the caller, >= kHdrWords words).  scratch >= kTreeScratchInts ints.
// plan_block() = build_tree(lit) + build_tree(dist) + plan_block_finish(), serially; k_plan runs the same steps with the
// order-free ones spread over its warps.
B200Z_HDN void plan_block_finish(const int *lit_freqs, const int *dist_freqs, int extra_bits, int stored_ok, int storedLength,
                                 int lastBlock, int lit_nc, const int *lit_blc, int dist_nc, const int *dist_blc, uint8_t *lit_len,
                                 uint16_t *lit_codes, uint8_t *dist_len, uint16_t *dist_codes, uint32_t *hdr_words, int *scratch,
                                 BlockPlan &plan);

B200Z_HDN void plan_block(const int *lit_freqs, const int *dist_freqs, int extra_bits, int stored_ok, int storedLength,
                          int lastBlock, uint8_t *lit_len, uint16_t *lit_codes, uint8_t *dist_len, uint16_t *dist_codes,
                          uint32_t *hdr_words, int *scratch, BlockPlan &plan) {
	int lit_blc[15], dist_blc[15];
	int lit_nc = build_tree(lit_freqs, kLiteralNum, 257, 15, lit_len, lit_blc, scratch);
	int dist_nc = build_tree(dist_freqs, kDistNum, 1, 15, dist_len, dist_blc, scratch);
	plan_block_finish(lit_freqs, dist_freqs, extra_bits, stored_ok, storedLength, lastBlock, lit_nc, lit_blc, dist_nc, dist_blc,
	                  lit_len, lit_codes, dist_len, dist_codes, hdr_words, scratch, plan);
}

B200Z_HDN void plan_block_finish(const int *lit_freqs, const int *dist_freqs, int extra_bits, int stored_ok, int storedLength,
                                 int lastBlock, int lit_nc, const int *lit_blc, int dist_nc, const int *dist_blc, uint8_t *lit_len,
                                 uint16_t *lit_codes, uint8_t *dist_len, uint16_t *dist_codes, uint32_t *hdr_words, int *scratch,
                                 BlockPlan &plan) {
	int bl_blc[7];
	int bl_freqs[kBitlenNum];
	uint8_t bl_len[kBitlenNum];
	uint16_t bl_codes[kBitlenNum];
	for (int i = 0; i < kBitlenNum; i++) bl_freqs[i] = 0;
	walk_code_lengths(lit_len, lit_nc, [&](int s) { bl_freqs[s]++; }, [&](int, int) {});
	walk_code_lengths(dist_len, dist_nc, [&](int s) { bl_freqs[s]++; }, [&](int, int) {});
	build_tree(bl_freqs, kBitlenNum, 4, 7, bl_len, bl_blc, scratch);
	int blTreeCodes = 4;
	for (int i = 18; i > blTreeCodes; i--) {
		if (bl_len[bl_order(i)] > 0) blTreeCodes = i + 1;
	}
	int opt_len = 14 + blTreeCodes * 3 + extra_bits;
	for (int i = 0; i < kBitlenNum; i++) opt_len += bl_freqs[i] * bl_len[i];
	for (int i = 0; i < kLiteralNum; i++) opt_len += lit_freqs[i] * lit_len[i];
	for (int i = 0; i < kDistNum; i++) opt_len += dist_freqs[i] * dist_len[i];
	int static_len = extra_bits;
	for (int i = 0; i < kLiteralNum; i++) static_len += lit_freqs[i] * static_llen(i);
	for (int i = 0; i < kDistNum; i++) static_len += dist_freqs[i] * 5;
	plan.lit_numCodes = lit_nc;
	plan.dist_numCodes = dist_nc;
	plan.blTreeCodes = blTreeCodes;
	plan.static_len = static_len;
	plan.type = block_type(stored_ok, storedLength, opt_len, static_len);
	if (opt_len >= static_len) opt_len = static_len;
	plan.opt_len = opt_len;
	if (plan.type == 0) {
		plan.hdr_bits = 3;
		plan.body_bits = 0;
		hdr_words[0] = (uint32_t)((0 << 1) + (lastBlock ? 1 : 0));
	} else if (plan.type == 1) {
		plan.hdr_bits = 3;
		plan.body_bits = (uint32_t)static_len;
		hdr_words[0] = (uint32_t)((1 << 1) + (lastBlock ? 1 : 0));
		for (int i = 0; i < kLiteralNum; i++) {
			lit_len[i] = (uint8_t)static_llen(i);
			lit_codes[i] = (uint16_t)static_lcode(i);
		}
		for (int i = 0; i < kDistNum; i++) {
			dist_len[i] = 5;
			dist_codes[i] = (uint16_t)static_dcode(i);
		}
	} else {
		// SendAllTrees (:676-696)
		build_codes(bl_len, bl_blc, 7, kBitlenNum, bl_codes); // blTree.numCodes is irrelevant: all 19 get codes
		build_codes(lit_len, lit_blc, 15, lit_nc, lit_codes);
		build_codes(dist_len, dist_blc, 15, dist_nc, dist_codes);
		BitSink sink{hdr_words, 0};
		sink.put((uint32_t)((2 << 1) + (lastBlock ? 1 : 0)), 3);
		sink.put((uint32_t)(lit_nc - 257), 5);
		sink.put((uint32_t)(dist_nc - 1), 5);
		sink.put((uint32_t)(blTreeCodes - 4), 4);
		for (int rank = 0; rank < blTreeCodes; rank++) sink.put(bl_len[bl_order(rank)], 3);
		walk_code_lengths(lit_len, lit_nc, [&](int s) { sink.put(bl_codes[s], bl_len[s]); },
		                  [&](int v, int nb) { sink.put((uint32_t)v, nb); });
		walk_code_lengths(dist_len, dist_nc, [&](int s) { sink.put(bl_codes[s], bl_len[s]); },
		                  [&](int v, int nb) { sink.put((uint32_t)v, nb); });
		plan.hdr_bits = sink.nbits;
		// body = literal/length + distance code bits + extra bits (dyn_len minus the 14 + 3*blTreeCodes + bl part)
		int body = extra_bits;
		for (int i = 0; i < kLiteralNum; i++) body += lit_freqs[i] * lit_len[i];
		for (int i = 0; i < kDistNum; i++) body += dist_freqs[i] * dist_len[i];
		plan.body_bits = (uint32_t)body;
	}
}

// Code word of one tallied symbol under the block's tables (CompressBlock :701-757): up to 48 bits, LSB first.
B200Z_HD void encode_symbol(uint32_t sym, const uint16_t *lit_codes, const uint8_t *lit_len, const uint16_t *dist_codes,
                            const uint8_t *dist_len, uint64_t &bits, int &nbits) {
	uint32_t dist = sym_dist(sym);
	if (dist == 0) {
		bits = lit_codes[sym & 0xFF];
		nbits = lit_len[sym & 0xFF];
		return;
	}
	int litlen = (int)(sym & 0xFF);
	int lc = lcode(litlen);
	uint64_t acc = lit_codes[lc];
	int nb = lit_len[lc];
	int eb = lcode_extra_bits(lc);
	if (eb) {
		acc |= (uint64_t)(litlen & ((1 << eb) - 1)) << nb;
		nb += eb;
	}
	int dm1 = (int)dist - 1;
	int dc = dcode(dm1);
	acc |= (uint64_t)dist_codes[dc] << nb;
	nb += dist_len[dc];
	eb = dcode_extra_bits(dc);
	if (eb) {
		acc |= (uint64_t)(dm1 & ((1 << eb) - 1)) << nb;
		nb += eb;
	}
	bits = acc;
	nbits = nb;
}

// TallyDist's extra_bits contribution (:899-913)
B200Z_HD int tally_extra_bits(int lc, int dc) {
	int e = 0;
	if (lc >= 265 && lc < 285) e += (lc - 261) / 4;
	if (dc >= 4) e += dc / 2 - 1;
	return e;
}

} // namespace b200z
