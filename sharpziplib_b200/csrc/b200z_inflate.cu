// b200z_inflate.cu -- the sm_90a DEFLATE decompressor.
//
// Replaces the reference's Inflater mode machine and its helpers:
//   Inflater.Decode / DecodeHuffman          Zip/Compression/Inflater.cs:429-552, :283-386
//   InflaterDynHeader.CreateStateMachine     Zip/Compression/InflaterDynHeader.cs:42-120
//   InflaterHuffmanTree.BuildTree/GetSymbol  Zip/Compression/InflaterHuffmanTree.cs:87-169, :181-235
//   OutputWindow.Write/Repeat/CopyStored     Zip/Compression/Streams/OutputWindow.cs:35-122
//   StreamManipulator (bit reader)           Zip/Compression/Streams/StreamManipulator.cs:31-298
//
// One warp per stream.  Block headers (and the code tables they describe) are handled by lane 0.  Inside a Huffman
// block the warp works in ROUNDS over the next 32 x kSubBits bits of input, staged in shared memory:
//   1. every lane decodes (count only) the symbols of its own sub-chunk, lane 0 from the true bit position, the others
//      from a guessed one; each lane then takes the previous lane's exit position as its entry and decodes again if that
//      changed.  Huffman streams re-synchronise within a few symbols, so this settles after ~2 passes; by induction the
//      first k+1 lanes are exact after k hand-offs, so it is exact after at most 32.
//   2. a prefix sum of the produced byte counts gives every lane its output position; a final decode pass stores the
//      literals into a 64 KiB output ring in shared memory (the reference's OutputWindow, doubled so that a whole round
//      fits behind 32 KiB of history) and records the back-references (position, length, distance) per lane.
//   3. back-references are resolved in stream order, each copied by the whole warp inside the ring with
//      OutputWindow.Repeat's byte-serial overlap rule (byte k comes from source byte k mod distance).
//   4. the round's bytes are flushed from the ring to the output buffer with coalesced vector stores.
// The ring starts zeroed: a distance reaching before the start of the stream reads zeros, which is what a fresh
// reference window holds (trap T13: the reference does not check distances).
#include <cstdlib>
#include <cstring>

#include <cuda_pipeline.h>

#include "b200z_internal.cuh"

namespace b200z {

constexpr int kLitRoot = 10, kDistRoot = 9;

// Inflater.cs:39-68
__constant__ uint16_t c_cplens[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_cplext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_cpdist[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_cpdext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_meta_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15}; // InflaterDynHeader.cs:24

// status detail codes (bits 8..15 of the per-stream status word); messages in INTEGRATION.md
enum {
	D_NONE = 0,
	D_BLOCK_TYPE = 1,   // "Unknown block type"                      Inflater.cs:486
	D_STORED_LEN = 2,   // "broken uncompressed block"               Inflater.cs:511
	D_REP_LEN = 3,      // "Illegal rep length code"                 Inflater.cs:325
	D_REP_DIST = 4,     // "Illegal rep dist code"                   Inflater.cs:358
	D_CODELEN0 = 5,     // "Encountered invalid codelength 0"        InflaterHuffmanTree.cs:192
	D_HDR_RANGE = 6,    // ValueOutOfRangeException                  InflaterDynHeader.cs:50-52
	D_HDR_REPEAT0 = 7,  // "Cannot repeat previous code length ..."  InflaterDynHeader.cs:83
	D_HDR_OVERRUN = 8,  // "Cannot repeat code lengths past ..."     InflaterDynHeader.cs:106
	D_HDR_NO_EOB = 9,   // "... end-of-block code missing"           InflaterDynHeader.cs:114
	D_OVERSUBSCRIBED = 10, // the reference indexes out of range here; reported as a data error
	// framing (zlib: Inflater.DecodeHeader / DecodeChksum; gzip: GZipInputStream.ReadHeader / ReadFooter)
	D_ADLER = 11,        // "Adler chksum doesn't match"               Inflater.cs:413
	D_GZIP_CRC = 12,     // "GZIP crc sum mismatch"                    GzipInputStream.cs:338
	D_GZIP_ISIZE = 13,   // "Number of bytes mismatch in footer"       GzipInputStream.cs:350
	D_GZIP_MAGIC1 = 14,  // "Error GZIP header, first magic byte ..."  GzipInputStream.cs:194
	D_GZIP_MAGIC2 = 15,  // "... second magic byte doesn't match"      GzipInputStream.cs:200
	D_GZIP_METHOD = 16,  // "... data not in deflate format"          GzipInputStream.cs:209
	D_GZIP_FLAGS = 17,   // "Reserved flag bits in GZIP header != 0"   GzipInputStream.cs:222
	D_GZIP_HCRC = 18,    // "Header CRC value mismatch"                GzipInputStream.cs:305
	D_ZLIB_HCHECK = 19,  // "Header checksum illegal"                  Inflater.cs:224
	D_ZLIB_METHOD = 20,  // "Compression Method unknown"               Inflater.cs:229
	D_NEED_DICT = 22     // FDICT set and the plan holds no dictionary for the stream (Inflater.IsNeedingDictionary)
};

// decode table entry: nb[0..3] | kind[4..7] | extra[8..11] | base[16..31]
enum { K_INVALID = 0, K_LIT = 1, K_EOB = 2, K_LEN = 3, K_LONG = 4, K_ILLEGAL = 5, K_DIST = 6 };
__device__ __forceinline__ uint32_t mk_entry(uint32_t nb, uint32_t kind, uint32_t extra, uint32_t base) {
	return nb | (kind << 4) | (extra << 8) | (base << 16);
}
__device__ __forceinline__ uint32_t litlen_entry(uint32_t sym, uint32_t nb) {
	if (sym < 256) return mk_entry(nb, K_LIT, 0, sym);
	if (sym == 256) return mk_entry(nb, K_EOB, 0, 0);
	if (sym - 257 >= 29) return mk_entry(nb, K_ILLEGAL, 0, 0);
	return mk_entry(nb, K_LEN, c_cplext[sym - 257], c_cplens[sym - 257]);
}
__device__ __forceinline__ uint32_t dist_entry(uint32_t sym, uint32_t nb) {
	if (sym >= 30) return mk_entry(nb, K_ILLEGAL, 0, 0);
	return mk_entry(nb, K_DIST, c_cpdext[sym], c_cpdist[sym]);
}

struct Canon { // canonical-code bookkeeping for codes longer than the root table
	uint16_t first[16], count[16], offs[16];
};

struct __align__(16) InfShared {
	uint32_t lit[1 << kLitRoot];
	uint32_t dist[1 << kDistRoot];
	uint32_t meta[128];
	uint16_t lit_sorted[288];
	uint16_t dist_sorted[32];
	Canon lit_c, dist_c;
	uint8_t lens[320];
	uint16_t tok_len[32];
	uint16_t tok_val[32];
};

// Builds a root table of `R` bits + canonical side tables from code lengths (InflaterHuffmanTree.BuildTree :87-169
// computes the same canonical assignment).  kind: 0 litlen, 1 dist, 2 meta (19 code-length symbols, 7-bit root, no
// long codes possible).  Returns 0 or a detail code.  Executed by one lane.
__device__ int build_table(const uint8_t *lens, int nsym, int R, uint32_t *tab, uint16_t *sorted, Canon *cn, int kind) {
	uint32_t count[16], next[16];
	for (int i = 0; i < 16; i++) count[i] = 0;
	for (int s = 0; s < nsym; s++) count[lens[s]]++;
	count[0] = 0;
	int left = 1;
	for (int L = 1; L <= 15; L++) {
		left = (left << 1) - (int)count[L];
		if (left < 0) return D_OVERSUBSCRIBED;
	}
	uint32_t code = 0, off = 0;
	for (int L = 1; L <= 15; L++) {
		next[L] = code;
		if (cn) {
			cn->first[L] = (uint16_t)code;
			cn->count[L] = (uint16_t)count[L];
			cn->offs[L] = (uint16_t)off;
		}
		if (L > R) off += count[L];
		code = (code + count[L]) << 1;
	}
	const int size = 1 << R;
	for (int i = 0; i < size; i++) tab[i] = 0;
	for (int s = 0; s < nsym; s++) {
		const int L = lens[s];
		if (!L) continue;
		const uint32_t c = next[L]++;
		const uint32_t rev = __brev(c) >> (32 - L);
		if (L <= R) {
			const uint32_t e = kind == 0 ? litlen_entry(s, L) : (kind == 1 ? dist_entry(s, L) : mk_entry(L, K_LIT, 0, s));
			for (uint32_t i = rev; i < (uint32_t)size; i += (1u << L)) tab[i] = e;
		} else {
			sorted[cn->offs[L] + (c - cn->first[L])] = (uint16_t)s;
			tab[rev & (size - 1)] = mk_entry(0, K_LONG, 0, 0);
		}
	}
	return 0;
}

struct BitReader {
	const uint32_t *words; // 4-byte aligned stream base
	uint64_t bb;
	uint32_t bc;     // valid bits in bb
	uint32_t widx;   // next word to load
	uint32_t nwords; // words that hold stream bytes (the last one is masked)
	uint32_t nbytes;
	uint64_t consumed; // bits handed out so far
	__device__ __forceinline__ void refill() {
		if (bc <= 32) {
			uint32_t w = 0;
			if (widx < nwords) {
				w = __ldg(words + widx);
				if (widx == nwords - 1 && (nbytes & 3)) w &= (1u << (8 * (nbytes & 3))) - 1u;
			}
			++widx;
			bb |= (uint64_t)w << bc;
			bc += 32;
		}
	}
	__device__ __forceinline__ uint32_t peek(int n) const { return (uint32_t)bb & ((1u << n) - 1u); }
	__device__ __forceinline__ void drop(int n) {
		bb >>= n;
		bc -= n;
		consumed += n;
	}
	__device__ __forceinline__ uint32_t get(int n) {
		refill();
		uint32_t v = peek(n);
		drop(n);
		return v;
	}
	__device__ __forceinline__ bool overrun() const { return consumed > 8ull * nbytes; }
};

// decodes one symbol of a tree with long-code fallback; returns the entry (nb already dropped) or 0 when invalid
__device__ __forceinline__ uint32_t decode_sym(BitReader &br, const uint32_t *tab, int R, const uint16_t *sorted,
                                               const Canon &cn, int kind) {
	br.refill();
	uint32_t e = tab[(uint32_t)br.bb & ((1u << R) - 1u)];
	const uint32_t k = (e >> 4) & 15;
	if (k != K_LONG) {
		if (k != K_INVALID) br.drop(e & 15);
		return e;
	}
	const uint32_t x = __brev((uint32_t)br.bb) >> 17; // next 15 stream bits, first bit most significant
	for (int L = R + 1; L <= 15; L++) {
		const uint32_t c = x >> (15 - L);
		const uint32_t idx = c - cn.first[L];
		if (idx < cn.count[L]) {
			const uint32_t s = sorted[cn.offs[L] + idx];
			br.drop(L);
			return kind == 0 ? litlen_entry(s, L) : dist_entry(s, L);
		}
	}
	return 0;
}

constexpr int kSubBits = 512;                 // input bits per lane per round
constexpr int kRoundWords = 32 * kSubBits / 32;  // 512 words
constexpr int kInWords = kRoundWords + 8;        // + slack for the last symbol's overshoot
// Lane l reads around word 16 l: laid out linearly, all 32 lanes would hit two shared-memory banks (16-way conflicts on
// every peek).  One pad word per 16 moves lane l to 17 l.
__device__ __forceinline__ uint32_t in_slot(uint32_t i) { return i + (i >> 4); }
constexpr int kInSlots = kInWords + kInWords / 16 + 1;
constexpr int kLaneOutCap = 512;                 // output bytes a lane may produce per round
constexpr int kRing = 65536;                     // output ring: 32 KiB of history + the two rounds the consumer warps hold (2 x 32 x kLaneOutCap)
constexpr int kMList = 32;                       // back-references a lane may record per round

enum { F_EOB = 1, F_ERR = 2, F_OVERRUN = 4, F_DEAD = 8 };

// The round's input lives in shared memory, so a lane needs no bit buffer: the 32 bits that start at any bit position
// are two words and a funnel shift away.  The decode state of a lane is just its bit position.
__device__ __forceinline__ uint32_t peek32(const uint32_t *w, uint32_t pos) {
	const uint32_t i = pos >> 5;
	return __funnelshift_r(w[in_slot(i)], w[in_slot(i + 1)], pos & 31u); // i + 1 < kInWords is guaranteed by the staging slack
}

// decodes one symbol of a tree at `v` (the next 32 stream bits); returns the entry and the code length in nb
__device__ __forceinline__ uint32_t lane_decode_sym(uint32_t v, const uint32_t *tab, int R, const uint16_t *sorted,
                                                    const Canon &cn, int kind, uint32_t &nb) {
	const uint32_t e = tab[v & ((1u << R) - 1u)];
	const uint32_t k = (e >> 4) & 15;
	nb = e & 15;
	if (k != K_LONG) return e;
	const uint32_t x = __brev(v) >> 17; // next 15 stream bits, first bit most significant
	for (int L = R + 1; L <= 15; L++) {
		const uint32_t c = x >> (15 - L);
		const uint32_t idx = c - cn.first[L];
		if (idx < cn.count[L]) {
			const uint32_t s = sorted[cn.offs[L] + idx];
			nb = (uint32_t)L;
			return kind == 0 ? litlen_entry(s, L) : dist_entry(s, L);
		}
	}
	nb = 0;
	return 0;
}

// Per-lane decode state of one span (the symbols that START in [entry, limit), relative bit positions).
struct Span {
	uint32_t pos, o, nm, fl, det;
};

// Decodes ONE symbol of the span.  Returns true while the lane should keep going.  The callers drive it in a
// warp-synchronous loop (all lanes step together and re-converge every iteration) -- a per-lane `while` loop leaves the
// 32 lanes diverged for the whole span, which ncu showed as 3.6 active threads per instruction.
// FINAL = false: counts only.  FINAL = true: literals go to the ring at output position obase + o, back-references
// to ml[0 .. nm).  A symbol that does not fit the lane's caps, or that needs bits past the end of the input, is not
// consumed (pos stays at its first bit).
template <bool FINAL>
__device__ __forceinline__ bool span_step(const InfShared &sh, const uint32_t *words, Span &s, uint32_t limit,
                                          uint32_t end_rel, uint8_t *win, uint32_t obase, uint2 *ml) {
	const uint32_t spos = s.pos;
	if (spos >= limit) return false;
	uint32_t v = peek32(words, spos);
	uint32_t nb;
	const uint32_t e = lane_decode_sym(v, sh.lit, kLitRoot, sh.lit_sorted, sh.lit_c, 0, nb);
	const uint32_t k = (e >> 4) & 15;
	if (k == K_LIT) {
		if (spos + nb > end_rel) { s.fl |= F_OVERRUN; return false; }
		if (s.o + 1 > (uint32_t)kLaneOutCap) return false;
		if (FINAL) win[(obase + s.o) & (uint32_t)(kRing - 1)] = (uint8_t)(e >> 16);
		++s.o;
		s.pos = spos + nb;
		return true;
	}
	if (k == K_LEN) {
		// length code (<= 15 bits) + extra (<= 5) fit the first peek; the distance code + extra (<= 28) a second one
		const uint32_t xb = (e >> 8) & 15;
		const uint32_t len = (e >> 16) + ((v >> nb) & ((1u << xb) - 1u));
		uint32_t pos = spos + nb + xb;
		v = peek32(words, pos);
		uint32_t dnb;
		const uint32_t de = lane_decode_sym(v, sh.dist, kDistRoot, sh.dist_sorted, sh.dist_c, 1, dnb);
		const uint32_t dk = (de >> 4) & 15;
		if (dk != K_DIST) {
			// (InflaterHuffmanTree.GetSymbol :181-235: an entry without a code is diagnosed once 9 bits can be peeked, a code for an
			// illegal symbol once its own bits are there; with fewer bits the decoder waits for more input)
			if (pos + (dk == K_ILLEGAL ? dnb : 9u) > end_rel) s.fl |= F_OVERRUN;
			else { s.fl |= F_ERR; s.det = dk == K_ILLEGAL ? D_REP_DIST : D_CODELEN0; }
			return false;
		}
		const uint32_t dxb = (de >> 8) & 15;
		const uint32_t dist = (de >> 16) + ((v >> dnb) & ((1u << dxb) - 1u));
		pos += dnb + dxb;
		if (pos > end_rel) { s.fl |= F_OVERRUN; return false; }
		if (s.o + len > (uint32_t)kLaneOutCap || s.nm >= (uint32_t)kMList) return false;
		if (FINAL) ml[s.nm] = make_uint2(obase + s.o, len | (dist << 16));
		++s.nm;
		s.o += len;
		s.pos = pos;
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

// What warp A hands to warp B for one round.
struct RoundInfo {
	uint32_t entry[32];  // true entry bit position of every lane (relative to the round's first staged bit)
	uint32_t obytes[32]; // bytes each lane produces (0 beyond the last live lane)
	uint32_t nmatch[32]; // back-references each lane records
	uint64_t opos;       // output position of the round
	uint32_t end_rel;
	int lastlane;
	int tab;             // which InfShared the round's block uses
	int valid;
};

struct __align__(16) InfBlockShared {
	InfShared sh[2];          // code tables, double buffered: A may build the next block's while B still decodes
	uint32_t in[2][kInSlots]; // staged input words (in_slot layout), double buffered
	RoundInfo ri[3];          // round r lives in ri[r % 3]: written by A, read by B1 one iteration later and by B2 two later
	uint32_t rs_out[3], rs_nm[3]; // per round, from B1 to B2: bytes produced, back-references recorded
	__align__(16) uint8_t ring[kRing]; // ring[pos & 65535] = output byte `pos`; doubles as OutputWindow (Streams/OutputWindow.cs:15-23)
	__align__(16) uint2 mlist[2][32 * kMList]; // flat, in stream order: x = output position (low 32 bits), y = len | dist << 16
	int a_done;
};
constexpr int kInfSmem2 = (int)sizeof(InfBlockShared);

// Three warps per stream, one round apart each.  Warp A (producer): block headers, code tables, and the counted decode
// passes of round t (speculative lanes, exit -> entry hand-off until stable).  Warp B1: final decode pass of round t-1
// (literals into the ring, back-reference records into a list).  Warp B2: the copies of round t-2 and its flush.  One
// __syncthreads per round keeps them in step; a single warp per stream is latency bound (ncu: IPC 0.16), and with two
// warps the consumer (decode + copies + flush) was the longer half, so the stages overlap almost for free.
constexpr int kInfThreads = 96;
__global__ void __launch_bounds__(kInfThreads)
    k_inflate(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, const int64_t *__restrict__ in_off,
              const int64_t *__restrict__ in_len, const int64_t *__restrict__ out_off, const int64_t *__restrict__ out_cap,
              int nstreams, int64_t *__restrict__ out_len, int64_t *__restrict__ in_used, int32_t *__restrict__ status,
              const uint32_t *__restrict__ dict_len, const uint32_t *__restrict__ start_bit, const int32_t *__restrict__ pre,
              int64_t *__restrict__ restart, const int32_t *__restrict__ only) {
	extern __shared__ __align__(16) uint8_t smem_raw[];
	InfBlockShared &S = *reinterpret_cast<InfBlockShared *>(smem_raw);
	const int lane = threadIdx.x & 31;
	const bool isA = threadIdx.x < 32, isB1 = threadIdx.x >= 32 && threadIdx.x < 64;
	const int stream = blockIdx.x;
	if (stream >= nstreams) return;
	if (only && !only[stream]) return; // behind the block-parallel pipeline: only the streams it handed back (k_chain)
	if (pre && pre[stream] != B200Z_OK) { // the framing header was rejected (k_wrap_head): nothing to decode
		if (threadIdx.x == 0) {
			status[stream] = pre[stream];
			out_len[stream] = 0;
			if (in_used) in_used[stream] = 0;
			restart[2 * stream] = 0;
			restart[2 * stream + 1] = 0;
		}
		return;
	}
	uint8_t *dst = out + out_off[stream];
	const uint64_t cap = (uint64_t)out_cap[stream];
	const uint32_t *gwords = reinterpret_cast<const uint32_t *>(in + in_off[stream]);

	BitReader br; // warp A lane 0's header reader (global memory)
	br.words = gwords;
	br.nbytes = (uint32_t)in_len[stream];
	br.nwords = (br.nbytes + 3) >> 2;
	br.bb = 0;
	br.bc = 0;
	br.widx = 0;
	br.consumed = 0;
	const uint64_t total_bits = 8ull * br.nbytes;

	for (int i = threadIdx.x; i < kRing / 16; i += kInfThreads) reinterpret_cast<uint4 *>(S.ring)[i] = make_uint4(0, 0, 0, 0); // fresh window = zeros
	if (threadIdx.x == 0) {
		S.ri[0].valid = 0;
		S.ri[1].valid = 0;
		S.ri[2].valid = 0;
		S.a_done = 0;
	}
	__syncthreads();
	{
		// preset dictionary (Inflater.SetDictionary -> OutputWindow.CopyDict, OutputWindow.cs:151-171): its last <= 32768
		// bytes lie directly in front of the compressed data and become the window contents behind output position 0
		const uint32_t D = dict_len[stream];
		const uint8_t *dsrc = in + in_off[stream] - D;
		for (uint32_t i = threadIdx.x; i < D; i += kInfThreads) S.ring[(uint32_t)kRing - D + i] = dsrc[i];
		if (D) __syncthreads();
	}

	// ---- warp A state (uniform across the warp unless noted) ----
	uint64_t opos = 0;   // bytes produced by all rounds handed over so far
	uint64_t bitpos = start_bit ? start_bit[stream] : 0u; // true bit position of the next symbol / header (behind a framing header)
	int st = B200Z_OK, detail = 0;
	bool last = false, in_block = false, a_done = false, pending_stored = false;
	uint32_t stored_len = 0;
	// restart point: bit position of the last block header reached and the output position there.  A caller that only
	// has part of a stream (the Inflater handle between SetInput calls) decodes on from this header instead of from the
	// start: everything the decoder carries across a block boundary is the window (the output) and the bit position.
	uint64_t rs_bit = bitpos, rs_out = 0;
	int tab = 0, static_in = -1; // static_in: which table buffer currently holds the static tables (-1 none)

	for (uint32_t t = 0;; t++) {
		const int cur = (int)(t & 1), prv = cur ^ 1;                                   // input staging / match list buffers
		const int r0i = (int)(t % 3), r1i = (int)((t + 2) % 3), r2i = (int)((t + 1) % 3); // RoundInfo of rounds t, t-1, t-2
		if (isA) {
			// ============================ producer ============================
			int valid = 0;
			if (!a_done) {
				const bool b_busy = S.ri[r1i].valid != 0 || S.ri[r2i].valid != 0; // B1 / B2 still hold earlier rounds
				if (pending_stored) {
					if (!b_busy) {
						// ---- stored block: OutputWindow.CopyStored (:100-122); B is idle, so the ring and dst are ours
						const uint64_t ipos = bitpos >> 3;
						const uint64_t avail = ipos <= br.nbytes ? br.nbytes - ipos : 0;
						if (stored_len > avail) st = B200Z_E_NEED_INPUT;
						else if (opos + stored_len > cap) st = B200Z_E_NOMEM;
						if (st == B200Z_OK) {
							const uint8_t *src = in + in_off[stream] + ipos;
							for (uint32_t i = lane; i < stored_len; i += 32) {
								const uint8_t v = src[i];
								dst[opos + i] = v;
								S.ring[(uint32_t)(opos + i) & (uint32_t)(kRing - 1)] = v;
							}
							opos += stored_len;
							bitpos = 8ull * (ipos + stored_len);
							pending_stored = false;
						} else {
							a_done = true;
						}
					}
				} else {
					if (!in_block) {
						// ---- block header (lane 0) -------------------------------------------------------
						int btype = 0;
						const int ntab = tab ^ 1; // B may still be decoding the previous round with `tab`
						if (!last) {
							rs_bit = bitpos;
							rs_out = opos;
						}
						if (lane == 0) {
							// re-seat the header reader at the true bit position
							br.consumed = bitpos;
							br.widx = (uint32_t)(bitpos >> 5);
							br.bb = 0;
							br.bc = 0;
							const uint32_t sk = (uint32_t)(bitpos & 31);
							if (sk) {
								br.refill();
								br.bb >>= sk;
								br.bc -= sk;
							}
							if (last) {
								btype = -1; // Inflater.cs:443-449: raw mode stops right after the final block
							} else {
								const uint32_t hdr = br.get(3);
								if (br.overrun()) {
									st = B200Z_E_NEED_INPUT;
								} else {
									last = (hdr & 1) != 0;
									btype = (int)(hdr >> 1);
									InfShared &sh = S.sh[ntab];
									if (btype == 0) {
										// SkipToByteBoundary, LEN, NLEN (:509)
										br.drop(br.bc & 7);
										const uint32_t len = br.get(16);
										const uint32_t nlen = br.get(16);
										if (br.overrun()) st = B200Z_E_NEED_INPUT;
										else if (nlen != (len ^ 0xFFFFu)) { st = B200Z_E_DATA; detail = D_STORED_LEN; }
										stored_len = len;
									} else if (btype == 1) {
										if (static_in != ntab) {
											for (int i = 0; i < 144; i++) sh.lens[i] = 8;
											for (int i = 144; i < 256; i++) sh.lens[i] = 9;
											for (int i = 256; i < 280; i++) sh.lens[i] = 7;
											for (int i = 280; i < 288; i++) sh.lens[i] = 8;
											build_table(sh.lens, 288, kLitRoot, sh.lit, sh.lit_sorted, &sh.lit_c, 0);
											for (int i = 0; i < 32; i++) sh.lens[i] = 5;
											build_table(sh.lens, 32, kDistRoot, sh.dist, sh.dist_sorted, &sh.dist_c, 1);
											static_in = ntab;
										}
									} else if (btype == 2) {
										if (static_in == ntab) static_in = -1;
										// InflaterDynHeader.CreateStateMachine (:42-120)
										const int nlit = (int)br.get(5) + 257, ndist = (int)br.get(5) + 1, nmeta = (int)br.get(4) + 4;
										if (nlit > 286 || ndist > 30) { st = B200Z_E_DATA; detail = D_HDR_RANGE; }
										else {
											for (int i = 0; i < 19; i++) sh.lens[i] = 0;
											for (int i = 0; i < nmeta; i++) sh.lens[c_meta_order[i]] = (uint8_t)br.get(3);
											int d = build_table(sh.lens, 19, 7, sh.meta, nullptr, nullptr, 2);
											if (d) { st = B200Z_E_DATA; detail = d; }
											const int total = nlit + ndist;
											int idx = 0;
											while (st == B200Z_OK && idx < total) {
												br.refill();
												const uint32_t e = sh.meta[br.peek(7)];
												if (((e >> 4) & 15) == K_INVALID) { st = B200Z_E_DATA; detail = D_CODELEN0; break; }
												br.drop(e & 15);
												const int sym = (int)(e >> 16);
												if (sym < 16) {
													sh.lens[idx++] = (uint8_t)sym;
												} else {
													int rep;
													uint8_t v = 0;
													if (sym == 16) {
														if (idx == 0) { st = B200Z_E_DATA; detail = D_HDR_REPEAT0; break; }
														v = sh.lens[idx - 1];
														rep = 3 + (int)br.get(2);
													} else if (sym == 17) rep = 3 + (int)br.get(3);
													else rep = 11 + (int)br.get(7);
													if (idx + rep > total) { st = B200Z_E_DATA; detail = D_HDR_OVERRUN; break; }
													while (rep-- > 0) sh.lens[idx++] = v;
												}
												if (br.overrun()) { st = B200Z_E_NEED_INPUT; break; }
											}
											if (st == B200Z_OK && br.overrun()) st = B200Z_E_NEED_INPUT;
											if (st == B200Z_OK && sh.lens[256] == 0) { st = B200Z_E_DATA; detail = D_HDR_NO_EOB; }
											if (st == B200Z_OK) {
												uint8_t dl[32];
												for (int i = 0; i < ndist; i++) dl[i] = sh.lens[nlit + i];
												d = build_table(sh.lens, nlit, kLitRoot, sh.lit, sh.lit_sorted, &sh.lit_c, 0);
												if (!d) d = build_table(dl, ndist, kDistRoot, sh.dist, sh.dist_sorted, &sh.dist_c, 1);
												if (d) { st = B200Z_E_DATA; detail = d; }
											}
										}
									} else {
										st = B200Z_E_DATA;
										detail = D_BLOCK_TYPE;
									}
								}
							}
							// an error diagnosed from bits past the end of the input is "needs more input", not corrupt data
							if (st != B200Z_OK && br.overrun()) { st = B200Z_E_NEED_INPUT; detail = 0; }
						}
						st = __shfl_sync(0xffffffffu, st, 0);
						btype = __shfl_sync(0xffffffffu, btype, 0);
						last = __shfl_sync(0xffffffffu, (int)last, 0) != 0;
						static_in = __shfl_sync(0xffffffffu, static_in, 0);
						bitpos = __shfl_sync(0xffffffffu, (unsigned long long)br.consumed, 0);
						stored_len = __shfl_sync(0xffffffffu, stored_len, 0);
						__syncwarp();
						if (st != B200Z_OK || btype == -1) {
							a_done = true;
						} else if (btype == 0) {
							pending_stored = true; // copied in a later iteration, once B is idle
						} else {
							tab = ntab;
							in_block = true;
						}
					}
					if (in_block && !a_done) {
						// ---- one round: stage words, counted passes with exit -> entry hand-off ---------------------
						uint32_t *words = S.in[cur];
						const InfShared &sh = S.sh[tab];
						const uint32_t w0 = (uint32_t)(bitpos >> 5);
						for (int i = lane; i < kInWords; i += 32) {
							const uint32_t wi = w0 + (uint32_t)i;
							uint32_t v = 0;
							if (wi < br.nwords) {
								v = __ldg(gwords + wi);
								if (wi == br.nwords - 1 && (br.nbytes & 3)) v &= (1u << (8 * (br.nbytes & 3))) - 1u;
							}
							words[in_slot((uint32_t)i)] = v;
						}
						__syncwarp();
						const uint32_t r0 = (uint32_t)(bitpos & 31);
						const uint64_t remain = total_bits - ((uint64_t)w0 << 5);
						const uint32_t end_rel = remain > 0x7FFFFFFFull ? 0x7FFFFFFFu : (uint32_t)remain;
						const uint32_t limit = r0 + (uint32_t)(lane + 1) * kSubBits;
						uint32_t entry = r0 + (uint32_t)lane * kSubBits;
						uint32_t exitp = entry, obytes = 0, nmatch = 0, flags = 0, det = 0;
						bool changed = true, dead = false;
						for (int it = 0; it < 34; it++) {
							Span sp;
							bool act = changed && !dead;
							if (changed) {
								sp.o = 0;
								sp.nm = 0;
								sp.fl = dead ? (uint32_t)F_DEAD : 0u;
								sp.det = 0;
								sp.pos = entry;
							}
							while (__any_sync(0xffffffffu, act)) {
								if (act) act = span_step<false>(sh, words, sp, limit, end_rel, nullptr, 0, nullptr);
								__syncwarp();
							}
							if (changed) {
								exitp = sp.pos;
								obytes = sp.o;
								nmatch = sp.nm;
								flags = sp.fl;
								det = sp.det;
							}
							const uint32_t pe = __shfl_up_sync(0xffffffffu, exitp, 1);
							const uint32_t pf = __shfl_up_sync(0xffffffffu, flags, 1);
							changed = false;
							if (lane > 0) {
								const bool nd = pf != 0; // the previous lane ended the block, failed or is dead itself
								changed = (pe != entry) || (nd != dead);
								entry = pe;
								dead = nd;
							}
							if (!__any_sync(0xffffffffu, changed)) break;
						}
						// lanes up to and including the first one that stopped the block are exact; the rest are dead
						const uint32_t stopmask = __ballot_sync(0xffffffffu, (flags & (F_EOB | F_ERR | F_OVERRUN)) != 0);
						const int lastlane = stopmask ? (__ffs(stopmask) - 1) : 31;
						if (lane > lastlane) { obytes = 0; nmatch = 0; }
						uint32_t tot = obytes;
						for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
						const uint32_t lflags = __shfl_sync(0xffffffffu, flags, lastlane);
						const uint32_t ldet = __shfl_sync(0xffffffffu, det, lastlane);
						const uint32_t lexit = __shfl_sync(0xffffffffu, exitp, lastlane);
						if (opos + tot > cap) {
							st = B200Z_E_NOMEM;
							a_done = true;
						} else {
							RoundInfo &ri = S.ri[r0i];
							ri.entry[lane] = entry;
							ri.obytes[lane] = obytes;
							ri.nmatch[lane] = nmatch;
							if (lane == 0) {
								ri.opos = opos;
								ri.end_rel = end_rel;
								ri.lastlane = lastlane;
								ri.tab = tab;
							}
							valid = 1;
							opos += tot;
							bitpos = ((uint64_t)w0 << 5) + lexit;
							if (lflags & F_EOB) in_block = false;
							else if (lflags & F_OVERRUN) { st = B200Z_E_NEED_INPUT; a_done = true; }
							else if (lflags & F_ERR) { st = B200Z_E_DATA; detail = (int)ldet; a_done = true; }
							else if (tot == 0 && lexit == r0) { st = B200Z_E_INTERNAL; a_done = true; } // cannot happen: a symbol always fits
						}
					}
				}
			}
			if (lane == 0) {
				S.ri[r0i].valid = valid;
				S.a_done = a_done ? 1 : 0;
			}
		} else if (isB1) {
			// ============================ consumer, first half: final decode pass of round t-1 ============================
			const RoundInfo &ri = S.ri[r1i];
			if (ri.valid) {
				const InfShared &sh = S.sh[ri.tab];
				const uint32_t *words = S.in[prv];
				const uint32_t entry = ri.entry[lane], obytes = ri.obytes[lane], nmatch = ri.nmatch[lane];
				const uint64_t ropos = ri.opos;
				const int lastlane = ri.lastlane;
				const uint32_t end_rel = ri.end_rel;
				uint32_t incl = obytes, mincl = nmatch;
				for (int o = 1; o < 32; o <<= 1) {
					const uint32_t t1 = __shfl_up_sync(0xffffffffu, incl, o);
					const uint32_t t2 = __shfl_up_sync(0xffffffffu, mincl, o);
					if (lane >= o) { incl += t1; mincl += t2; }
				}
				const uint32_t round_out = __shfl_sync(0xffffffffu, incl, 31);
				const uint32_t total_m = __shfl_sync(0xffffffffu, mincl, 31);
				const uint32_t obase = (uint32_t)ropos + incl - obytes; // this lane's first output position (low 32 bits)
				// lane l's span ends where lane l + 1's nominal sub-chunk starts; r0 is lane 0's entry
				const uint32_t r0 = __shfl_sync(0xffffffffu, entry, 0);
				const uint32_t lim = r0 + (uint32_t)(lane + 1) * kSubBits;
				{
					Span sp;
					bool act = lane <= lastlane && obytes != 0;
					sp.o = 0;
					sp.nm = 0;
					sp.fl = 0;
					sp.det = 0;
					sp.pos = entry;
					uint2 *ml = S.mlist[prv] + (mincl - nmatch);
					while (__any_sync(0xffffffffu, act)) {
						if (act) act = span_step<true>(sh, words, sp, lim, end_rel, S.ring, obase, ml);
						__syncwarp();
					}
				}
				__syncwarp();
				if (lane == 0) {
					S.rs_out[r1i] = round_out;
					S.rs_nm[r1i] = total_m;
				}
			}
		} else {
			// ============================ consumer, second half: copies and flush of round t-2 ============================
			const RoundInfo &ri = S.ri[r2i];
			if (ri.valid) {
				const uint64_t ropos = ri.opos;
				const uint32_t round_out = S.rs_out[r2i], total_m = S.rs_nm[r2i];
				const uint2 *mlist = S.mlist[cur]; // round t-2 has the parity of t
				// ---- back-references in stream order (OutputWindow.Repeat :63-92) ----------------------------------
				// Four matches per step, each copied by a group of 8 lanes, when none of them reads bytes another match
				// of the same step writes; otherwise the step's matches are copied one after another by the whole warp.
				// All sources are in the ring (distance <= 32768 < ring size - round size); byte k comes from source byte
				// k mod distance, which only reads bytes that were final before this match.
				{
					const int grp = lane >> 3, sub = lane & 7;
					for (uint32_t k0 = 0; k0 < total_m; k0 += 4) {
						const uint32_t mi = k0 + (uint32_t)grp;
						const bool have = mi < total_m;
						const uint2 m = have ? mlist[mi] : make_uint2(0u, 0u);
						const uint32_t mo = m.x, mlen = m.y & 0xFFFFu, mdist = m.y >> 16;
						const uint32_t step_lo = __shfl_sync(0xffffffffu, mo, 0); // first destination byte of this step
						// a later match of the step depends on the step if its source reaches step_lo or beyond
						const uint32_t shi = mo - mdist + (mlen < mdist ? mlen : mdist);
						const bool dep = have && grp > 0 && (int32_t)(shi - step_lo) > 0;
						if (!__any_sync(0xffffffffu, dep)) {
							if (have) {
								const uint32_t sbase = mo - mdist;
								if (mdist >= mlen) {
									for (uint32_t k2 = sub; k2 < mlen; k2 += 8)
										S.ring[(mo + k2) & (uint32_t)(kRing - 1)] = S.ring[(sbase + k2) & (uint32_t)(kRing - 1)];
								} else {
									for (uint32_t k2 = sub; k2 < mlen; k2 += 8)
										S.ring[(mo + k2) & (uint32_t)(kRing - 1)] = S.ring[(sbase + k2 % mdist) & (uint32_t)(kRing - 1)];
								}
							}
							__syncwarp();
						} else {
							for (int g = 0; g < 4; g++) {
								const uint32_t gmo = __shfl_sync(0xffffffffu, mo, g * 8);
								const uint32_t gy = __shfl_sync(0xffffffffu, m.y, g * 8);
								const bool ghave = __shfl_sync(0xffffffffu, (int)have, g * 8) != 0;
								if (ghave) {
									const uint32_t glen = gy & 0xFFFFu, gdist = gy >> 16, gs = gmo - gdist;
									if (gdist >= glen) {
										for (uint32_t k2 = lane; k2 < glen; k2 += 32)
											S.ring[(gmo + k2) & (uint32_t)(kRing - 1)] = S.ring[(gs + k2) & (uint32_t)(kRing - 1)];
									} else {
										for (uint32_t k2 = lane; k2 < glen; k2 += 32)
											S.ring[(gmo + k2) & (uint32_t)(kRing - 1)] = S.ring[(gs + k2 % gdist) & (uint32_t)(kRing - 1)];
									}
								}
								__syncwarp();
							}
						}
					}
				}
				// ---- flush the round: ring[opos .. opos + round_out) -> dst, 16-byte vectors where aligned ------------
				{
					const uint64_t b0 = ropos, b1 = ropos + round_out;
					const uint64_t v0 = (b0 + 15) & ~15ull, v1 = b1 & ~15ull;
					if (v0 < v1) {
						for (uint64_t i = b0 + lane; i < v0; i += 32) dst[i] = S.ring[(uint32_t)i & (uint32_t)(kRing - 1)];
						for (uint64_t i = v0 + 16ull * lane; i < v1; i += 512)
							*reinterpret_cast<uint4 *>(dst + i) = *reinterpret_cast<const uint4 *>(S.ring + ((uint32_t)i & (uint32_t)(kRing - 1)));
						for (uint64_t i = v1 + lane; i < b1; i += 32) dst[i] = S.ring[(uint32_t)i & (uint32_t)(kRing - 1)];
					} else {
						for (uint64_t i = b0 + lane; i < b1; i += 32) dst[i] = S.ring[(uint32_t)i & (uint32_t)(kRing - 1)];
					}
				}
			}
		}
		__syncthreads();
		// (the three flags into registers, then a second barrier: warp A's next iteration overwrites them)
		const bool stop_now = S.a_done && !S.ri[r0i].valid && !S.ri[r1i].valid;
		__syncthreads();
		if (stop_now) break; // A has nothing more, B1 and B2 nothing left to take over
	}
	if (threadIdx.x == 0) {
		status[stream] = st | (detail << 8);
		out_len[stream] = (int64_t)opos;
		if (in_used) {
			uint64_t used = (bitpos + 7) >> 3; // n - RemainingInput (trap T14)
			if (used > br.nbytes) used = br.nbytes;
			in_used[stream] = (int64_t)used;
		}
		restart[2 * stream] = (int64_t)rs_bit;
		restart[2 * stream + 1] = (int64_t)rs_out;
	}
}

// ------------------------------------------------------------------------------------------------
// Framing around the raw stream, one thread per stream.  zlib: Inflater.DecodeHeader (:209-247) and DecodeChksum
// (:397-418); gzip: GZipInputStream.ReadHeader (:169-311) and ReadFooter (:313-357), one member per plan slot (a caller
// with multi-member input runs the rest again, in_used tells where it starts).
// ------------------------------------------------------------------------------------------------
__global__ void k_wrap_head(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                            const uint32_t *__restrict__ dict_len, int n, int wrap, uint32_t *__restrict__ start_bit,
                            int32_t *__restrict__ pre) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint8_t *p = in + in_off[i];
	const uint64_t len = (uint64_t)in_len[i];
	int st = B200Z_OK, det = 0;
	uint64_t pos = 0;
	if (wrap == B200Z_WRAP_ZLIB) {
		if (len < 2) st = B200Z_E_NEED_INPUT;
		else {
			const uint32_t header = ((uint32_t)p[0] << 8) | p[1];
			if (header % 31 != 0) { st = B200Z_E_DATA; det = D_ZLIB_HCHECK; }
			else if ((header & 0x0f00) != (8u << 8)) { st = B200Z_E_DATA; det = D_ZLIB_METHOD; }
			else {
				pos = 2;
				if (header & 0x0020) { // PRESET_DICT: DICTID follows (:185-203); the caller has checked it against its dictionary
					if (len < 6) st = B200Z_E_NEED_INPUT;
					else if (dict_len[i] == 0) { st = B200Z_E_DATA; det = D_NEED_DICT; }
					else pos = 6;
				}
			}
		}
	} else if (wrap == B200Z_WRAP_GZIP) {
		// header CRC over every header byte read (:190-283), byte at a time with the table-0 recurrence
		uint32_t crc = 0xFFFFFFFFu;
		auto upd = [&](uint32_t b) { crc = crc_table0_entry((crc ^ b) & 0xFFu) ^ (crc >> 8); };
		auto need = [&](uint64_t k) {
			if (pos + k > len) { st = B200Z_E_NEED_INPUT; return false; } // "EOS reading GZIP header"
			return true;
		};
		if (need(10)) {
			if (p[0] != 0x1F) { st = B200Z_E_DATA; det = D_GZIP_MAGIC1; }
			else if (p[1] != 0x8B) { st = B200Z_E_DATA; det = D_GZIP_MAGIC2; }
			else if (p[2] != 8) { st = B200Z_E_DATA; det = D_GZIP_METHOD; }
			else if (p[3] & 0xE0) { st = B200Z_E_DATA; det = D_GZIP_FLAGS; }
		}
		if (st == B200Z_OK) {
			const uint32_t flags = p[3];
			for (int k = 0; k < 10; k++) upd(p[k]);
			pos = 10;
			if (flags & 4) { // FEXTRA
				if (need(2)) {
					const uint32_t xlen = (uint32_t)p[pos] | ((uint32_t)p[pos + 1] << 8);
					upd(p[pos]);
					upd(p[pos + 1]);
					pos += 2;
					if (need(xlen)) {
						for (uint32_t k = 0; k < xlen; k++) upd(p[pos + k]);
						pos += xlen;
					}
				}
			}
			for (int field = 0; field < 2 && st == B200Z_OK; field++) { // FNAME, FCOMMENT: zero terminated
				if (!(flags & (field == 0 ? 8u : 16u))) continue;
				for (;;) {
					if (!need(1)) break;
					const uint32_t b = p[pos++];
					upd(b);
					if (b == 0) break;
				}
			}
			if (st == B200Z_OK && (flags & 2)) { // FHCRC: the reference reads it high byte first (:286-306)
				if (need(2)) {
					const uint32_t crcval = ((uint32_t)p[pos] << 8) | p[pos + 1];
					pos += 2;
					if (crcval != ((crc ^ 0xFFFFFFFFu) & 0xFFFFu)) { st = B200Z_E_DATA; det = D_GZIP_HCRC; }
				}
			}
		}
	}
	start_bit[i] = (uint32_t)(8u * pos);
	pre[i] = st | (det << 8);
}

__global__ void k_wrap_tail(const uint8_t *__restrict__ in, const int64_t *__restrict__ in_off, const int64_t *__restrict__ in_len,
                            int n, int wrap, int64_t *__restrict__ in_used, const int64_t *__restrict__ out_len,
                            const uint32_t *__restrict__ check, int32_t *__restrict__ status) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if ((status[i] & 0xFF) != B200Z_OK) return; // the stream did not end: nothing to compare
	const uint8_t *p = in + in_off[i];
	const uint64_t len = (uint64_t)in_len[i];
	uint64_t used = (uint64_t)in_used[i];
	const uint64_t want = wrap == B200Z_WRAP_ZLIB ? 4u : 8u;
	if (used + want > len) { // DecodeChksum waits for more input; "EOS reading GZIP footer"
		status[i] = B200Z_E_NEED_INPUT;
		in_used[i] = (int64_t)len;
		return;
	}
	const uint8_t *t = p + used;
	if (wrap == B200Z_WRAP_ZLIB) {
		const uint32_t theirs = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
		if (theirs != check[i]) status[i] = B200Z_E_DATA | (D_ADLER << 8);
	} else {
		const uint32_t crcval = (uint32_t)t[0] | ((uint32_t)t[1] << 8) | ((uint32_t)t[2] << 16) | ((uint32_t)t[3] << 24);
		const uint32_t total = (uint32_t)t[4] | ((uint32_t)t[5] << 8) | ((uint32_t)t[6] << 16) | ((uint32_t)t[7] << 24);
		if (crcval != check[i]) status[i] = B200Z_E_DATA | (D_GZIP_CRC << 8);
		else if (total != (uint32_t)((uint64_t)out_len[i] & 0xFFFFFFFFu)) status[i] = B200Z_E_DATA | (D_GZIP_ISIZE << 8);
	}
	in_used[i] = (int64_t)(used + want);
}

} // namespace b200z
#include "b200z_inflate_par.cuh"
namespace b200z {

// ------------------------------------------------------------------------------------------------
int inflate_plan_build(b200z_plan *p) {
	const int n = p->n;
	p->in_off.resize(n);
	p->out_off.resize(n);
	int64_t io = 0, oo = 0;
	const bool has_dict = !p->hist.empty();
	std::vector<int64_t> dev_off(n), dev_len(n);
	std::vector<uint32_t> dict32(n, 0u);
	for (int i = 0; i < n; i++) {
		if (p->in_len[i] < 0 || p->in_len[i] > 0xFFFF0000ll || p->out_cap[i] < 0) {
			set_error("stream %d: size out of range", i);
			return B200Z_E_ARG;
		}
		// slot: [pad][dictionary][compressed data], the compressed data 16-byte aligned; in_len[] counts dictionary + data
		const int64_t D = has_dict ? p->hist[i] : 0;
		const int64_t comp = io + align_up(D, 16);
		p->in_off[i] = comp - D;
		dev_off[i] = comp;
		dev_len[i] = p->in_len[i] - D;
		p->comp_off.push_back(comp);
		p->comp_cap.push_back(dev_len[i]);
		p->dict_cap.push_back(D);
		dict32[i] = (uint32_t)D;
		io = comp + align_up(dev_len[i] + 16, kAlign);
		io = align_up(io, kAlign);
		p->out_off[i] = oo;
		oo += align_up(p->out_cap[i] + 16, kAlign);
	}
	p->in_bytes = io;
	p->out_bytes = oo;
	Arena &ws = p->ws;
	p->o_in_off = ws.reserve(8ll * (n + 1));
	p->o_in_len = ws.reserve(8ll * (n + 1));
	p->o_out_off = ws.reserve(8ll * (n + 1));
	p->o_out_cap = ws.reserve(8ll * (n + 1));
	p->o_hist = ws.reserve(4ll * (n + 1));
	p->o_start_bit = ws.reserve(4ll * (n + 1));
	p->o_pre = ws.reserve(4ll * (n + 1));
	p->o_restart = ws.reserve(16ll * (n + 1));
	std::vector<CkTile> ck_tiles;
	if (p->wrap != B200Z_WRAP_RAW) {
		// checksum of the OUTPUT (Adler-32 for zlib, CRC-32 for gzip and raw+CRC): tiles over the capacities, the kernel takes
		// the real lengths from d_out_len
		checksum_tiles(p->out_cap.data(), n, ck_tiles, p->wrap == B200Z_WRAP_ZLIB ? 1 : 0, true);
		p->n_ck_tiles = (int)ck_tiles.size();
		p->o_ck_desc = ws.reserve((int64_t)sizeof(CkTile) * (ck_tiles.size() + 1));
		p->o_ck_acc = ws.reserve(16ll * (n + 1));
	}
	// ---- block-parallel pipeline: candidate windows, finder tiles, pools (b200z_inflate_par.cuh) ----
	{
		const char *mode = getenv("B200Z_INFLATE");
		p->inf_parallel = !(mode && strcmp(mode, "serial") == 0);
	}
	std::vector<uint32_t> win_base(n + 1, 0u), win_stream, match_cap(n, 0u);
	std::vector<FTile> ftiles;
	std::vector<int64_t> mt_off(n, 0);
	if (p->inf_parallel && n) {
		uint64_t nwin = 0, rounds = 0, bits = 0, mt = 0;
		for (int i = 0; i < n; i++) {
			const uint64_t len = (uint64_t)dev_len[i];
			win_base[i] = (uint32_t)nwin;
			const uint64_t w = len ? (len * 8 + kFWMask) >> kFWShift : 1;
			for (uint64_t k = 0; k < w; k++) win_stream.push_back((uint32_t)i);
			nwin += w;
			bits += len * 8;
			rounds += 4 * ((len * 8 + (uint64_t)kP1Threads * kSubBits - 1) / ((uint64_t)kP1Threads * kSubBits)) + 16;
			const uint32_t nw = (uint32_t)((len + 3) >> 2);
			for (uint32_t w0 = 0; w0 < nw; w0 += kFindTileWords) {
				FTile t;
				t.stream = (uint32_t)i;
				t.word0 = w0;
				t.nwords = nw - w0 < (uint32_t)kFindTileWords ? nw - w0 : (uint32_t)kFindTileWords;
				t.pad = 0;
				ftiles.push_back(t);
			}
			// a back-reference takes at least two bits of input and produces at least three bytes
			uint64_t mc = (uint64_t)p->out_cap[i] / 3 + 2;
			if (mc > 4 * len + 2) mc = 4 * len + 2;
			if (mc > 0x7FFFFFFFull) mc = 0x7FFFFFFFull;
			match_cap[i] = (uint32_t)mc;
			mt_off[i] = (int64_t)mt;
			mt += mc;
		}
		win_base[n] = (uint32_t)nwin;
		if (nwin + (uint64_t)n > 0x7FFFFFF0ull || rounds > 0x7FFFFFF0ull) {
			p->inf_parallel = false; // (beyond the 32-bit slot numbers: the serial kernel takes the plan)
		} else {
			p->nwin_total = (uint32_t)nwin;
			p->n_ftiles = (uint32_t)ftiles.size();
			p->fs_cap = (uint32_t)(bits / 256 + 1024 > 0x7FFFFFFFull ? 0x7FFFFFFFull : bits / 256 + 1024);
			p->round_cap = (uint32_t)((rounds + kRoundBatch - 1) / kRoundBatch * kRoundBatch);
			p->hdr_cap = p->round_cap / kRoundBatch;
			p->o_win_base = ws.reserve(4ll * (n + 1));
			p->o_win_stream = ws.reserve(4ll * (int64_t)nwin);
			p->o_cand = ws.reserve(4ll * (int64_t)nwin);
			p->o_ftiles = ws.reserve((int64_t)sizeof(FTile) * (int64_t)(ftiles.size() + 1));
			p->o_fs_list = ws.reserve(8ll * p->fs_cap);
			p->o_ctr = ws.reserve((int64_t)sizeof(PCounters));
			p->o_segs = ws.reserve((int64_t)sizeof(PSeg) * (int64_t)(nwin + n));
			p->o_seg_list = ws.reserve(4ll * (int64_t)(nwin + n));
			p->o_rounds = ws.reserve((int64_t)sizeof(PRound) * p->round_cap);
			p->o_hdrs = ws.reserve((int64_t)sizeof(PBlockHdr) * p->hdr_cap);
			p->o_mlist = ws.reserve((int64_t)sizeof(MatchTok) * (int64_t)mt);
			p->o_mt_off = ws.reserve(8ll * (n + 1));
			p->o_match_cap = ws.reserve(4ll * (n + 1));
			p->o_str_nm = ws.reserve(4ll * (n + 1));
			p->o_fallback = ws.reserve(4ll * (n + 1));
		}
	}
	int rc = ws.alloc();
	if (rc) return rc;
	if (n) {
		B200Z_CUDA(cudaMemcpy(ws.at<int64_t>(p->o_in_off), dev_off.data(), 8ll * n, cudaMemcpyHostToDevice));
		B200Z_CUDA(cudaMemcpy(ws.at<int64_t>(p->o_in_len), dev_len.data(), 8ll * n, cudaMemcpyHostToDevice));
		B200Z_CUDA(cudaMemcpy(ws.at<uint32_t>(p->o_hist), dict32.data(), 4ll * n, cudaMemcpyHostToDevice));
		if (!ck_tiles.empty())
			B200Z_CUDA(cudaMemcpy(ws.at<CkTile>(p->o_ck_desc), ck_tiles.data(), sizeof(CkTile) * ck_tiles.size(), cudaMemcpyHostToDevice));
		B200Z_CUDA(cudaMemcpy(ws.at<int64_t>(p->o_out_off), p->out_off.data(), 8ll * n, cudaMemcpyHostToDevice));
		B200Z_CUDA(cudaMemcpy(ws.at<int64_t>(p->o_out_cap), p->out_cap.data(), 8ll * n, cudaMemcpyHostToDevice));
		if (p->inf_parallel) {
			B200Z_CUDA(cudaMemcpy(ws.at<uint32_t>(p->o_win_base), win_base.data(), 4ll * (n + 1), cudaMemcpyHostToDevice));
			B200Z_CUDA(cudaMemcpy(ws.at<uint32_t>(p->o_win_stream), win_stream.data(), 4ll * win_stream.size(), cudaMemcpyHostToDevice));
			if (!ftiles.empty())
				B200Z_CUDA(cudaMemcpy(ws.at<FTile>(p->o_ftiles), ftiles.data(), sizeof(FTile) * ftiles.size(), cudaMemcpyHostToDevice));
			B200Z_CUDA(cudaMemcpy(ws.at<int64_t>(p->o_mt_off), mt_off.data(), 8ll * n, cudaMemcpyHostToDevice));
			B200Z_CUDA(cudaMemcpy(ws.at<uint32_t>(p->o_match_cap), match_cap.data(), 4ll * n, cudaMemcpyHostToDevice));
		}
	}
	B200Z_CUDA(cudaFuncSetAttribute(k_inflate, cudaFuncAttributeMaxDynamicSharedMemorySize, kInfSmem2));
	int extra = 0;
	if (p->inf_parallel && n) {
		B200Z_CUDA(cudaFuncSetAttribute(k_resolve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ResShared)));
		// (the decode kernels want many small CTAs per SM: ask for the largest shared-memory carve-out)
		B200Z_CUDA(cudaFuncSetAttribute(k_dec1, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
		B200Z_CUDA(cudaFuncSetAttribute(k_dec2, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
		B200Z_CUDA(cudaFuncSetAttribute(k_find, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
		B200Z_CUDA(cudaFuncSetAttribute(k_find3, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
		int dev = 0, sms = 1, occ1 = 1, occ2 = 1;
		B200Z_CUDA(cudaGetDevice(&dev));
		B200Z_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
		B200Z_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, k_dec1, kP1Threads, sizeof(Dec1Shared)));
		B200Z_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, k_dec2, kP1Threads, sizeof(Dec2Shared)));
		if (occ1 < 1) occ1 = 1;
		if (occ2 < 1) occ2 = 1;
		const int64_t slots = (int64_t)p->nwin_total + n, batches = p->round_cap / kRoundBatch;
		p->dec1_grid = (int)(slots < (int64_t)sms * occ1 ? slots : (int64_t)sms * occ1);
		p->dec2_grid = (int)(batches < (int64_t)sms * occ2 ? batches : (int64_t)sms * occ2);
		{
			const int64_t want = ((int64_t)p->fs_cap + 127) / 128;
			p->find3_grid = (int)(want < (int64_t)sms * 16 ? want : (int64_t)sms * 16);
		}
		extra = 7; // k_find, k_find3, k_seglist, k_dec1, k_chain, k_dec2, k_resolve (+ k_inflate for what they hand back)
	}
	p->launches = extra + (p->wrap == B200Z_WRAP_RAW ? 1 : (p->wrap == B200Z_WRAP_RAW_CRC32 ? 4 : 6));
	return B200Z_OK;
}

int inflate_plan_stats(b200z_plan *p, uint32_t *v, int32_t cap, cudaStream_t s) {
	uint32_t r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	if (p->inf_parallel && p->n) {
		PCounters c;
		std::vector<int32_t> fb((size_t)p->n);
		B200Z_CUDA(cudaMemcpyAsync(&c, p->ws.at<PCounters>(p->o_ctr), sizeof(c), cudaMemcpyDeviceToHost, s));
		B200Z_CUDA(cudaMemcpyAsync(fb.data(), p->ws.at<int32_t>(p->o_fallback), 4ull * p->n, cudaMemcpyDeviceToHost, s));
		B200Z_CUDA(cudaStreamSynchronize(s));
		r[0] = c.fs_count;
		r[1] = c.nseg;
		r[2] = c.round_top;
		r[3] = c.n_blocks;
		r[4] = c.n_rounds;
		r[5] = c.n_passes;
		for (int i = 0; i < p->n; i++) r[6] += fb[(size_t)i] != 0;
		r[7] = 1;
	}
	for (int i = 0; i < cap && i < 8; i++) v[i] = r[i];
	return B200Z_OK;
}

int inflate_plan_run(b200z_plan *p, const uint8_t *d_in, uint8_t *d_out, int64_t *d_out_len, int32_t *d_status,
                     uint32_t *d_check, int64_t *d_in_used, cudaStream_t s) {
	const Arena &ws = p->ws;
	const int n = p->n;
	if (n == 0) return B200Z_OK;
	p->ev_used = 0;
	const int wrap = p->wrap;
	const bool framed = wrap == B200Z_WRAP_ZLIB || wrap == B200Z_WRAP_GZIP;
	if (wrap != B200Z_WRAP_RAW && (!d_check || !d_in_used)) {
		set_error("inflate plans with framing or checksums need d_check and d_in_used");
		return B200Z_E_ARG;
	}
	const int64_t *in_off = ws.at<int64_t>(p->o_in_off), *in_len = ws.at<int64_t>(p->o_in_len);
	uint32_t *start_bit = (framed || p->has_start_bits) ? ws.at<uint32_t>(p->o_start_bit) : nullptr;
	int32_t *pre = framed ? ws.at<int32_t>(p->o_pre) : nullptr;
	if (framed) {
		p->mark(s, "k_wrap");
		k_wrap_head<<<(n + 127) / 128, 128, 0, s>>>(d_in, in_off, in_len, ws.at<uint32_t>(p->o_hist), n, wrap, start_bit, pre);
	}
	const uint32_t *dict_len = ws.at<uint32_t>(p->o_hist);
	const int64_t *out_off = ws.at<int64_t>(p->o_out_off), *out_cap = ws.at<int64_t>(p->o_out_cap);
	int64_t *restart = ws.at<int64_t>(p->o_restart);
	const int32_t *only = nullptr;
	if (p->inf_parallel) {
		PCounters *ctr = ws.at<PCounters>(p->o_ctr);
		uint32_t *cand = ws.at<uint32_t>(p->o_cand);
		const uint32_t *win_base = ws.at<uint32_t>(p->o_win_base);
		PSeg *segs = ws.at<PSeg>(p->o_segs);
		uint32_t *seg_list = ws.at<uint32_t>(p->o_seg_list);
		PRound *rounds = ws.at<PRound>(p->o_rounds);
		PBlockHdr *hdrs = ws.at<PBlockHdr>(p->o_hdrs);
		MatchTok *mlist = ws.at<MatchTok>(p->o_mlist);
		const int64_t *mt_off = ws.at<int64_t>(p->o_mt_off);
		uint32_t *str_nm = ws.at<uint32_t>(p->o_str_nm);
		int32_t *fallback = ws.at<int32_t>(p->o_fallback);
		unsigned long long *fs_list = ws.at<unsigned long long>(p->o_fs_list);
		p->mark(s, "k_find");
		B200Z_CUDA(cudaMemsetAsync(ctr, 0, sizeof(PCounters), s));
		B200Z_CUDA(cudaMemsetAsync(cand, 0xFF, 4ull * p->nwin_total, s));
		if (p->n_ftiles)
			k_find<<<p->n_ftiles, 256, 0, s>>>(d_in, in_off, in_len, ws.at<FTile>(p->o_ftiles), start_bit, pre, fs_list, ctr, p->fs_cap);
		p->mark(s, "k_find3");
		k_find3<<<p->find3_grid, 128, 0, s>>>(d_in, in_off, in_len, fs_list, ctr, p->fs_cap, win_base, cand);
		p->mark(s, "k_seglist");
		const uint32_t slots = p->nwin_total + (uint32_t)n;
		k_seglist<<<(slots + 255) / 256, 256, 0, s>>>(n, p->nwin_total, win_base, ws.at<uint32_t>(p->o_win_stream), cand, start_bit, pre, segs,
		                                            seg_list, ctr);
		p->mark(s, "k_dec1");
		k_dec1<<<p->dec1_grid, kP1Threads, sizeof(Dec1Shared), s>>>(d_in, in_off, in_len, segs, seg_list, ctr, win_base, cand, rounds,
		                                                             p->round_cap, hdrs, p->hdr_cap);
		p->mark(s, "k_chain");
		k_chain<<<(n + 127) / 128, 128, 0, s>>>(n, segs, win_base, in_len, out_cap, ws.at<uint32_t>(p->o_match_cap), pre, d_out_len, d_in_used,
		                                        d_status, restart, str_nm, fallback);
		p->mark(s, "k_dec2");
		k_dec2<<<p->dec2_grid, kP1Threads, sizeof(Dec2Shared), s>>>(d_in, d_out, in_off, in_len, out_off, segs, ctr, rounds, p->round_cap, hdrs,
		                                                             mlist, mt_off);
		p->mark(s, "k_resolve");
		k_resolve<<<n, kResThreads, sizeof(ResShared), s>>>(d_in, d_out, in_off, out_off, dict_len, d_out_len, str_nm, fallback, mlist, mt_off, n);
		only = fallback;
	}
	p->mark(s, "k_inflate");
	k_inflate<<<n, kInfThreads, kInfSmem2, s>>>(d_in, d_out, in_off, in_len, out_off, out_cap, n, d_out_len, d_in_used, d_status, dict_len,
	                                           start_bit, pre, restart, only);
	if (wrap != B200Z_WRAP_RAW) {
		p->mark(s, "checksum");
		int rc = checksum_launch(wrap == B200Z_WRAP_ZLIB ? 1 : 0, d_out, ws.at<int64_t>(p->o_out_off), d_out_len, n,
		                         ws.at<CkTile>(p->o_ck_desc), p->n_ck_tiles, ws.at<unsigned long long>(p->o_ck_acc), d_check, 1, s);
		if (rc) return rc;
		if (framed) k_wrap_tail<<<(n + 127) / 128, 128, 0, s>>>(d_in, in_off, in_len, n, wrap, d_in_used, d_out_len, d_check, d_status);
	}
	p->mark(s, "end");
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

} // namespace b200z
