// b200z_handles.cu -- the streaming handles of the C-ABI (include/b200z.h), which mirror Deflater.cs / Inflater.cs member
// for member, and the Deflater sets, which run many Deflater streams through the same host path.  Each handle runs its
// plans synchronously from host buffers through one Staging (b200z_host.cuh), and so does a set.
#include <algorithm>
#include <cstring>

#include "b200z_host.cuh"

namespace b200z {

// ---- small host helpers ----------------------------------------------------------------------------
struct HostBits { // carries the sub-byte tail of a flushed stream on the host (PendingBuffer's `bits`, :23-24)
	uint32_t bits = 0;
	int count = 0;
	void put(std::vector<uint8_t> &out, uint32_t v, int n) {
		bits |= v << count;
		count += n;
		while (count >= 8) {
			out.push_back((uint8_t)bits);
			bits >>= 8;
			count -= 8;
		}
	}
	void align(std::vector<uint8_t> &out) {
		if (count > 0) out.push_back((uint8_t)bits);
		bits = 0;
		count = 0;
	}
};

void zlib_header(int level, uint8_t h[2], bool preset_dict) { // Deflater.cs:436-464 (trap T11)
	int header = (8 + (7 << 4)) << 8;
	int level_flags = (level - 1) >> 1;
	if (level_flags < 0 || level_flags > 3) level_flags = 3;
	header |= level_flags << 6;
	if (preset_dict) header |= 0x20; // DeflaterConstants.PRESET_DICT
	header += 31 - (header % 31);
	h[0] = (uint8_t)(header >> 8);
	h[1] = (uint8_t)header;
}

const char *inflate_detail_msg(int detail) {
	switch (detail) {
	case 1: return "Unknown block type";
	case 2: return "broken uncompressed block";
	case 3: return "Illegal rep length code";
	case 4: return "Illegal rep dist code";
	case 5: return "Encountered invalid codelength 0";
	case 6: return "ValueOutOfRangeException: dynamic header code count";
	case 7: return "Cannot repeat previous code length when no other code length has been read";
	case 8: return "Cannot repeat code lengths past total number of data code lengths";
	case 9: return "Inflater dynamic header end-of-block code missing";
	case 10: return "Code lengths oversubscribed";
	case 11: return "Adler chksum doesn't match";
	case 12: return "GZIP crc sum mismatch";
	case 13: return "Number of bytes mismatch in footer";
	case 14: return "Error GZIP header, first magic byte doesn't match";
	case 15: return "Error GZIP header,  second magic byte doesn't match";
	case 16: return "Error GZIP header, data not in deflate format";
	case 17: return "Reserved flag bits in GZIP header != 0";
	case 18: return "Header CRC value mismatch";
	case 19: return "Header checksum illegal";
	case 20: return "Compression Method unknown";
	case 22: return "Needs a preset dictionary";
	default: return "corrupt deflate data";
	}
}

std::string lzw_detail_msg(int32_t status, uint32_t value) {
	char b[160];
	switch ((status >> 8) & 0xFF) {
	case 32: snprintf(b, sizeof b, "Wrong LZW header. Magic bytes don't match. 0x%02x 0x%02x", value >> 8, value & 0xFF); break;
	case 33: snprintf(b, sizeof b, "Stream compressed with %u bits, but decompression can only handle 16 bits.", value); break;
	case 34: snprintf(b, sizeof b, "Unsupported bits set in the header."); break;
	case 35: snprintf(b, sizeof b, "corrupt input: %u > 255", value); break;
	case 36: snprintf(b, sizeof b, "corrupt input: code=%u, freeEnt=%u", value >> 16, value & 0xFFFF); break;
	default: snprintf(b, sizeof b, "LZW stream: the reference fails with a non-SharpZip exception (status detail %d)", (status >> 8) & 0xFF);
	}
	return b;
}

// One run of a handle's single-stream plan on the legacy default stream; returns with the run's metadata in st.h and the
// produced bytes in st.hout at the stream's out_off.  `in` is the handle's own pageable copy of the input.
static int handle_run(b200z_plan *plan, Staging &st, const uint8_t *in, const uint32_t *check_seed) {
	int rc = st.ensure(plan, false);
	if (!rc) rc = stage_run(plan, st, &in, false, check_seed, 0, 0, nullptr);
	if (rc) return rc;
	B200Z_CUDA(cudaStreamSynchronize(0));
	return streams_down(plan, st, nullptr, 0);
}

// =====================================================================================================
// Deflater streams: the Deflater handle and the Deflater set share one host path
// =====================================================================================================
constexpr b200z_parse_entry kCleanEntry = {0, kMinMatch - 1, 0};

// What one Deflater stream carries between device runs, whoever drives it (a handle, or a stream of a set).
struct StreamCarry {
	// what the engine's window has seen so far, cut to its last 32768 bytes (preset dictionary, then every compressed
	// segment); hist_mask flags the positions InsertString never saw (the last two of the dictionary / of each segment)
	std::vector<uint8_t> history, hist_mask;
	int64_t window_seen = 0; // dictionary bytes kept + TotalIn: the SlideWindow phase of the next segment
	bool started = false;    // an earlier segment (possibly empty) has been emitted
	std::vector<uint8_t> input; // everything SetInput handed over and not yet compressed
	// the parse state the next run starts from (levels 5-9), and the bytes at the front of `input` that the last open run
	// saw but left behind its cut
	b200z_parse_entry entry = kCleanEntry;
	int64_t carried = 0;
	// levels 0-4 depend on the call pattern (trap T9) and keep engine state across Flush() and cuts: the sizes of the SetInput
	// calls in `input` (behind a cut the first is the rest of the call the cut fell into), whether Deflate() was called behind
	// the last of them, and what the engines carry
	std::vector<int64_t> chunks;
	bool undrained = false;
	b200z_stored_state sstate = {1, 1, 0, 0}; // level 0 (DeflateStored; a fresh engine: strstart = blockStart = 1)
	DevBuf fstate;                            // levels 1-4 (DeflateFast: head[], prev[], scalars), on the device
	std::vector<uint8_t> pending; // produced bytes not yet handed out
	size_t pending_pos = 0;
	HostBits tail;                // sub-byte tail carried between device runs
	int64_t total_in = 0;
	uint32_t check = 1;           // the running Adler-32 (zlib) or CRC-32 (gzip, raw + CRC-32)
	void reset(uint32_t check0) { // (keeps the device buffer)
		history.clear();
		hist_mask.clear();
		window_seen = 0;
		started = false;
		input.clear();
		entry = kCleanEntry;
		carried = 0;
		chunks.clear();
		undrained = false;
		sstate = b200z_stored_state{1, 1, 0, 0};
		pending.clear();
		pending_pos = 0;
		tail = HostBits();
		total_in = 0;
		check = check0;
	}
};

static void carry_remember(StreamCarry *c, const uint8_t *seg, size_t len, size_t uninserted) {
	// append a dictionary/segment to the carried window image
	c->history.insert(c->history.end(), seg, seg + len);
	c->hist_mask.insert(c->hist_mask.end(), len, 0);
	for (size_t k = 0; k < uninserted && k < len; k++) c->hist_mask[c->hist_mask.size() - 1 - k] = 1;
	if (c->history.size() > 32768) {
		const size_t cut = c->history.size() - 32768;
		c->history.erase(c->history.begin(), c->history.begin() + (ptrdiff_t)cut);
		c->hist_mask.erase(c->hist_mask.begin(), c->hist_mask.begin() + (ptrdiff_t)cut);
	}
	c->window_seen += (int64_t)len;
}

// The bytes an open run may take: levels 0-4 whole SetInput calls whose Deflate() already ran (a call that Flush() /
// Finish() follows directly stays with the closing run, b200z_history.undrained_last), levels 5-9 all of `input`.
static int64_t open_run_avail(const StreamCarry *c, int level, int32_t *ncalls) {
	*ncalls = (int32_t)c->chunks.size() - ((level <= 4 && c->undrained && !c->chunks.empty()) ? 1 : 0);
	if (level >= 5) return (int64_t)c->input.size();
	int64_t avail = 0;
	for (int32_t k = 0; k < *ncalls; k++) avail += c->chunks[(size_t)k];
	return avail;
}

// The length of an open run that takes the carried bytes plus at most `most` more of `avail` (> most).  It is longer than a
// block can be, so it always ends in a cut and no run is repeated on the same bytes.  Levels 0-4 take enough whole calls to
// close a block, however long the last one is; *ncalls becomes the number taken.
static int64_t open_run_len(const StreamCarry *c, int level, int64_t avail, int64_t most, int32_t *ncalls) {
	const int64_t len = std::min<int64_t>(avail, c->carried + most);
	if (level >= 5) return len;
	int64_t sum = 0;
	int32_t k = 0;
	// (more than one block's reach behind the carried bytes: the run closes a block)
	const int64_t least = c->carried + (int64_t)kBlockSyms * kMaxMatch + kMaxMatch + kMinMatch + 1;
	while (k < *ncalls && (sum < least || sum + c->chunks[(size_t)k] <= len)) sum += c->chunks[(size_t)k++];
	*ncalls = k;
	return sum;
}

// One device run of the next segment of k streams of one level / strategy / end mode, as one plan: segments_begin builds
// the plan and enqueues the upload and the kernels on `cs`; segments_end waits for them, reads the cuts of an open run,
// carries each stream's running checksum over the bytes its run covered and appends the produced bytes to its `pending`.
// A run synchronises `cs` twice: once for the run's lengths and cuts, once for the produced bytes and checksums.
// wrap is B200Z_WRAP_RAW, _ZLIB (the checksum is an Adler-32) or _RAW_CRC32 (a CRC-32).
struct SegmentRun {
	int level = 6, strategy = 0, wrap = B200Z_WRAP_RAW, end_mode = B200Z_END_FINISH;
	std::vector<StreamCarry *> s;
	std::vector<int64_t> len;   // per stream: the first len[i] bytes of its input (levels 0-4: its first calls[i] SetInput calls)
	std::vector<int32_t> calls;
	b200z_plan *plan = nullptr;
	std::vector<b200z_stored_state> sbefore; // level 0: each state as the plan rebases it
	SegmentRun() = default;
	SegmentRun(const SegmentRun &) = delete;
	~SegmentRun() { b200z_plan_destroy(plan); }
	void add(StreamCarry *c, int64_t n, int32_t ncalls) {
		s.push_back(c);
		len.push_back(n);
		calls.push_back(ncalls);
	}
};

static int segments_begin(SegmentRun &r, Staging &st, cudaStream_t cs) {
	const int k = (int)r.s.size();
	const bool open = r.end_mode == B200Z_END_NONE;
	bool any_started = false, any_hist = false;
	for (const StreamCarry *c : r.s) {
		any_started |= c->started;
		any_hist |= !c->history.empty();
	}
	// A fresh stream next to continuing ones continues from nothing: no history, the fresh engine state
	const int kind = any_started ? B200Z_HIST_CONTINUE : (any_hist ? B200Z_HIST_DICTIONARY : B200Z_HIST_NONE);
	std::vector<int64_t> H((size_t)k), pos_base((size_t)k);
	std::vector<int32_t> bit_base((size_t)k), undrained((size_t)k);
	std::vector<const uint8_t *> mask((size_t)k), inp((size_t)k);
	std::vector<const int64_t *> chunk_ptr((size_t)k);
	std::vector<void *> fstate_ptr((size_t)k);
	std::vector<b200z_stored_state> sstate((size_t)k);
	std::vector<uint32_t> seed((size_t)k);
	std::vector<b200z_parse_entry> entry((size_t)k);
	std::vector<std::vector<uint8_t>> slot((size_t)k);
	r.sbefore.resize((size_t)k);
	for (int i = 0; i < k; i++) {
		StreamCarry *c = r.s[(size_t)i];
		if (kind == B200Z_HIST_CONTINUE && !c->started && !c->history.empty()) {
			set_error("a stream with a preset dictionary cannot start in a run with continuing streams");
			return B200Z_E_INTERNAL;
		}
		H[(size_t)i] = (int64_t)c->history.size();
		pos_base[(size_t)i] = c->window_seen;
		bit_base[(size_t)i] = c->tail.count;
		mask[(size_t)i] = c->hist_mask.data();
		chunk_ptr[(size_t)i] = c->chunks.data();
		undrained[(size_t)i] = (c->undrained && r.calls[(size_t)i] == (int32_t)c->chunks.size() && r.calls[(size_t)i] > 0 && !open) ? 1 : 0;
		if (r.level >= 1 && r.level <= 4) {
			int rc = c->fstate.ensure((size_t)b200z_engine_state_bytes());
			if (rc) return rc;
			fstate_ptr[(size_t)i] = c->fstate.p;
			if (kind == B200Z_HIST_CONTINUE && !c->started) { // DeflateFast as the constructor leaves it (fe_init)
				const FastCarry fresh = {1, 1, 0, 0, kMinMatch - 1, 0, 0u, 0u};
				B200Z_CUDA(cudaMemsetAsync(c->fstate.p, 0, 131072, cs));
				B200Z_CUDA(cudaMemcpyAsync(c->fstate.p + 131072, &fresh, sizeof fresh, cudaMemcpyHostToDevice, cs));
			}
		}
		sstate[(size_t)i] = c->sstate;
		// level 0: the state as the plan rebases it, for the bytes a closing run takes (see stored_run)
		r.sbefore[(size_t)i] = c->sstate;
		if (c->started) carry_rebase(r.sbefore[(size_t)i].slides, r.sbefore[(size_t)i].input_off);
		seed[(size_t)i] = c->check;
		entry[(size_t)i] = c->entry;
		inp[(size_t)i] = c->input.data();
		if (H[(size_t)i]) {
			std::vector<uint8_t> &v = slot[(size_t)i];
			v.reserve((size_t)(H[(size_t)i] + r.len[(size_t)i]));
			v.insert(v.end(), c->history.begin(), c->history.end());
			v.insert(v.end(), c->input.begin(), c->input.begin() + r.len[(size_t)i]);
			inp[(size_t)i] = v.data();
		}
	}
	b200z_history hs;
	memset(&hs, 0, sizeof hs);
	if (r.level <= 4) {
		hs.chunk_count = r.calls.data();
		hs.chunk_len = chunk_ptr.data();
		hs.undrained_last = undrained.data();
		if (r.level == 0) hs.stored_state = sstate.data();
		else hs.engine_state = fstate_ptr.data();
	}
	hs.kind = kind;
	hs.check_seeded = 1;
	hs.hist_len = H.data();
	hs.pos_base = pos_base.data();
	hs.bit_base = bit_base.data();
	hs.hist_mask = mask.data();
	int rc = b200z_deflate_plan_create_ex(k, r.len.data(), r.level, r.strategy, r.wrap, r.end_mode,
	                                      (kind != B200Z_HIST_NONE || r.level <= 4) ? &hs : nullptr, &r.plan);
	if (rc) return rc;
	if (r.level == 0) // (the plan wrote the state behind this segment when it was created)
		for (int i = 0; i < k; i++) r.s[(size_t)i]->sstate = sstate[(size_t)i];
	if (r.level >= 5 && (rc = b200z_deflate_plan_set_entry(r.plan, entry.data()))) return rc;
	// a plan with history continues the running checksum (hs.check_seeded)
	if ((rc = st.ensure(r.plan, false))) return rc;
	return stage_run(r.plan, st, inp.data(), false, (kind != B200Z_HIST_NONE && r.wrap != B200Z_WRAP_RAW && !open) ? seed.data() : nullptr,
	                 cs, cs, nullptr);
}

static int segments_end(SegmentRun &r, Staging &st, cudaStream_t cs) {
	const int k = (int)r.s.size();
	const bool open = r.end_mode == B200Z_END_NONE;
	B200Z_CUDA(cudaStreamSynchronize(cs));
	const PipeMeta &m = st.h;
	for (int i = 0; i < k; i++)
		if ((m.status[i] & 0xFF) != B200Z_OK) {
			set_error("device deflate failed with status %d", m.status[i] & 0xFF);
			return m.status[i] & 0xFF;
		}
	std::vector<int64_t> covered(r.len); // bytes of input each run is done with
	std::vector<b200z_parse_entry> next((size_t)k, kCleanEntry);
	std::vector<int32_t> cut_call((size_t)k, 0);
	std::vector<uint32_t> ck; // open runs: the running checksums behind the covered bytes
	int rc = B200Z_OK;
	if (open) {
		rc = b200z_deflate_plan_get_cut(r.plan, covered.data(), r.level >= 5 ? next.data() : nullptr, cs);
		if (!rc && r.level <= 4) rc = b200z_deflate_plan_get_cut_call(r.plan, cut_call.data(), cs);
		if (rc) return rc;
		for (int i = 0; i < k; i++)
			if (covered[(size_t)i] <= 0) { // (a run of more than 16384 * 258 + 262 bytes always closes a block)
				set_error("open run of %lld bytes closed no block", (long long)r.len[(size_t)i]);
				return B200Z_E_INTERNAL;
			}
		if (r.wrap != B200Z_WRAP_RAW) {
			// the checksums go on over the covered bytes, read from the copy of the input the run left on the device; the
			// values come back with the produced bytes (streams_down synchronises once for both)
			ck.resize((size_t)k);
			std::vector<int64_t> off((size_t)k);
			for (int i = 0; i < k; i++) {
				ck[(size_t)i] = r.s[(size_t)i]->check;
				off[(size_t)i] = b200z_plan_data_offset(r.plan, i);
			}
			B200Z_CUDA(cudaMemcpyAsync(st.d.check, ck.data(), 4ull * k, cudaMemcpyHostToDevice, cs));
			if ((rc = b200z_checksum_batch_device(r.wrap == B200Z_WRAP_ZLIB ? 1 : 0, st.din.p, off.data(), covered.data(), k, st.d.check, cs)))
				return rc;
			B200Z_CUDA(cudaMemcpyAsync(ck.data(), st.d.check, 4ull * k, cudaMemcpyDeviceToHost, cs));
		}
	}
	if ((rc = streams_down(r.plan, st, nullptr, cs))) return rc;
	for (size_t i = 0; i < ck.size(); i++) r.s[i]->check = ck[i];
	for (int i = 0; i < k; i++) {
		StreamCarry *c = r.s[(size_t)i];
		const int64_t len = r.len[(size_t)i], cov = covered[(size_t)i];
		const uint8_t *o = st.hout.p + r.plan->out_off[(size_t)i];
		const int64_t bits = m.in_used[i]; // deflate plans report the exact bit length here (bit_base included)
		const int64_t whole = bits >> 3;
		std::vector<uint8_t> seg(o, o + ((bits + 7) >> 3));
		if (!seg.empty()) seg[0] |= (uint8_t)c->tail.bits; // the carried sub-byte tail completes the first byte
		c->pending.insert(c->pending.end(), seg.begin(), seg.begin() + (ptrdiff_t)whole);
		// PendingBuffer keeps the sub-byte tail in `bits` until later writes complete the byte (:168-189)
		c->tail.count = (int)(bits & 7);
		c->tail.bits = c->tail.count ? (seg[(size_t)whole] & ((1u << c->tail.count) - 1u)) : 0u;
		if (r.end_mode == B200Z_END_FINISH) c->tail.align(c->pending); // FINISHING_STATE: AlignToByte (:507)
		if (r.wrap != B200Z_WRAP_RAW && !open) c->check = m.check[i];
		// (level 0: Finish() behind an undrained SetInput can end the stream before all input is taken, see stored_run;
		// the data starts strstart - block_start bytes in front of the state's input_off)
		const b200z_stored_state &sb = r.sbefore[(size_t)i];
		c->total_in += (r.level == 0 && !open) ? (int64_t)(uint32_t)(c->sstate.input_off - sb.input_off) + (sb.strstart - sb.block_start) : cov;
		c->started = true;
		// every position in front of a cut went through InsertString; a flush leaves the last two out
		carry_remember(c, c->input.data(), (size_t)cov, open ? 0 : 2);
		c->input.erase(c->input.begin(), c->input.begin() + cov);
		c->entry = next[(size_t)i];
		c->carried = len - cov;
		if (!open) {
			c->chunks.clear();
			c->undrained = false;
		} else if (r.level <= 4) {
			// the next run's schedule: the rest of the call the cut fell into, then the calls behind it
			int64_t end = 0;
			for (int32_t j = 0; j <= cut_call[(size_t)i]; j++) end += c->chunks[(size_t)j];
			c->chunks.erase(c->chunks.begin(), c->chunks.begin() + cut_call[(size_t)i]);
			c->chunks[0] = end - cov;
		}
	}
	return B200Z_OK;
}

// Finish() right behind a completed Flush(): every block and the sync padding are out, Finish adds the final empty block:
// levels 1-9 FlushBlock on an empty buffer = static header 011 + EOB 0000000 = value 3 in 10 bits (DeflaterEngine.cs:750-768);
// level 0 an empty stored block 01 00 00 FF FF (:614-649)
static void final_empty_block(StreamCarry *c, int level) {
	if (level == 0) {
		const uint8_t e5[5] = {1, 0, 0, 0xFF, 0xFF};
		c->pending.insert(c->pending.end(), e5, e5 + 5);
	} else {
		c->tail.put(c->pending, 3, 10);
		c->tail.align(c->pending);
	}
}

// behind the final block: zlib's Adler-32, big endian (Deflater.cs:509-514); gzip's CRC-32 and ISIZE = TotalIn & 0xFFFFFFFF,
// little endian (GZipOutputStream.GetFooter, :315-337); nothing for a raw stream
static void stream_trailer(StreamCarry *c, int wrap) {
	if (wrap == B200Z_WRAP_ZLIB) {
		for (int sh = 24; sh >= 0; sh -= 8) c->pending.push_back((uint8_t)(c->check >> sh));
	} else if (wrap == B200Z_WRAP_GZIP) {
		const uint32_t isz = (uint32_t)((uint64_t)c->total_in & 0xFFFFFFFFull);
		for (int sh = 0; sh < 32; sh += 8) c->pending.push_back((uint8_t)(c->check >> sh));
		for (int sh = 0; sh < 32; sh += 8) c->pending.push_back((uint8_t)(isz >> sh));
	}
}

// =====================================================================================================
// Streaming handles
// =====================================================================================================
// A long stream is compressed in open runs (B200Z_END_NONE) of this many new bytes, plus what the run in front left behind
// its cut: a plan's workspace grows with its input (about 3.7 GB for 256 MiB at levels 5-9), the host holds no more than
// that, and the output flows while input arrives.  A segment up to this size runs as one plan, as it always has.
constexpr int64_t kOpenRunBytes = 256ll << 20;

struct DeflaterH {
	int level = 6, strategy = 0;
	bool raw = false;
	// Deflater.cs state bits (:96-110)
	bool flushing = false, finishing = false, finished = false;
	bool header_done = false;
	bool flushed_once = false; // a sync flush has been emitted and nothing was compressed since
	bool dict_set = false, deflate_called = false;
	uint32_t dict_adler = 0;
	bool draining = false; // the output of an open run is still being handed out
	int64_t total_out = 0;
	StreamCarry s;
	Staging st;
};

static void deflater_header(DeflaterH *d) {
	if (!d->header_done && !d->raw) {
		uint8_t hd[2];
		zlib_header(d->level, hd, d->dict_set);
		d->s.pending.push_back(hd[0]);
		d->s.pending.push_back(hd[1]);
		if (d->dict_set) { // DICTID = Adler-32 of the whole dictionary, MSB first (:455-461)
			for (int sh = 24; sh >= 0; sh -= 8) d->s.pending.push_back((uint8_t)(d->dict_adler >> sh));
		}
	}
	d->header_done = true;
}

// compresses the first `len` bytes of the input (levels 0-4: the first n_chunks SetInput calls) as the next segment of the
// stream, in a plan of its own on the legacy default stream; END_FLUSH keeps the stream open and may end inside a byte;
// END_NONE writes the blocks that closed and keeps the bytes behind them for the next run
static int deflater_run_device(DeflaterH *d, int end_mode, int64_t len, int32_t n_chunks) {
	SegmentRun r;
	r.level = d->level;
	r.strategy = d->strategy;
	r.wrap = d->raw ? B200Z_WRAP_RAW : B200Z_WRAP_ZLIB;
	r.end_mode = end_mode;
	r.add(&d->s, len, n_chunks);
	int rc = segments_begin(r, d->st, 0);
	return rc ? rc : segments_end(r, d->st, 0);
}

// While more than one run's worth of input is buffered, the front of it is compressed in open runs and their output is due
// at once.  Each run takes the bytes its predecessor left behind the cut plus at most kOpenRunBytes more.
static int deflater_open_runs(DeflaterH *d) {
	for (;;) {
		int32_t ncalls = 0;
		const int64_t avail = open_run_avail(&d->s, d->level, &ncalls);
		if (avail <= kOpenRunBytes) return B200Z_OK;
		const int64_t len = open_run_len(&d->s, d->level, avail, kOpenRunBytes, &ncalls);
		if (d->s.pending_pos == d->s.pending.size()) {
			d->s.pending.clear();
			d->s.pending_pos = 0;
		}
		deflater_header(d);
		int rc = deflater_run_device(d, B200Z_END_NONE, len, ncalls);
		if (rc) return rc;
		d->draining = true;
	}
}

// ---- Deflater set ------------------------------------------------------------------------------------
// n Deflater streams of one level / strategy / wrap, driven together.  A write appends every stream's input as
// DeflaterOutputStream.Write hands it over (SetInput, then Deflate() until it needs input); then the streams with enough
// buffered run their open runs, the streams that flush their flushes and those that finish their finishes, each group in
// as few plans as kSetPlanBytes allows, one after the other on the set's CUDA stream.  A stream with no Flush() / Finish()
// due runs an open run once it holds kSetRunBytes beyond what it carries, and the run takes at most kSetRunBytes more than
// that (levels 0-4 end a run at a SetInput call, so it may take the rest of the call it reaches into).  kSetRunBytes is more
// than the 16384 * 258 + 262 bytes after which a run at levels 0-4 always closes a block.
// A plan's device workspace grows with its input (at levels 5-9 about 14 bytes per input byte), so the streams of one
// group are split into plans of at most kSetPlanBytes of input (history included; a stream longer than that runs alone):
// 256 streams due at once, about 256 x 8.5 MiB at most, take two or three plans, whatever the number of streams.
// (The CPU test tier builds the kernels on the CUDA emulator with smaller values, for small data.)
#ifndef B200Z_SET_RUN_BYTES
#define B200Z_SET_RUN_BYTES 4456448 // 4.25 MiB
#endif
#ifndef B200Z_SET_PLAN_BYTES
#define B200Z_SET_PLAN_BYTES (1ll << 30)
#endif
constexpr int64_t kSetRunBytes = B200Z_SET_RUN_BYTES;
constexpr int64_t kSetPlanBytes = B200Z_SET_PLAN_BYTES;

struct SetStream : StreamCarry {
	bool header_done = false, flushed_once = false, finished = false;
};

} // namespace b200z

struct b200z_deflate_streams {
	int device = -1, level = 6, strategy = 0, wrap = B200Z_WRAP_ZLIB;
	std::vector<b200z::SetStream> s;
	b200z::Staging st; // grows to the largest plan, at most kSetPlanBytes of input and its output bound, until destroy
	cudaStream_t cs = nullptr;
	int broken = 0; // a run failed: the streams' state is not what their output says, no more writes
	int64_t stats[4] = {0, 0, 0, 0}; // b200z_deflate_streams_stats
};

namespace b200z {

static void set_header(const b200z_deflate_streams *S, SetStream *c) {
	if (c->header_done) return;
	if (S->wrap == B200Z_WRAP_ZLIB) {
		uint8_t hd[2];
		zlib_header(S->level, hd);
		c->pending.insert(c->pending.end(), hd, hd + 2);
	} else if (S->wrap == B200Z_WRAP_GZIP) {
		// GZipOutputStream's header (GzipOutputStream.cs:339-375) with MTIME 0 and no FNAME, as the pipelines write it
		const uint8_t h[10] = {0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF};
		c->pending.insert(c->pending.end(), h, h + 10);
	}
	c->header_done = true;
}

struct SetDue { // a stream's next segment: its first len bytes, in its first `calls` SetInput calls
	SetStream *c;
	int64_t len;
	int32_t calls;
};

// runs the segments of one end mode in plans of at most kSetPlanBytes of input each
static int set_plans(b200z_deflate_streams *S, int end_mode, const std::vector<SetDue> &due) {
	for (size_t a = 0; a < due.size();) {
		SegmentRun r;
		r.level = S->level;
		r.strategy = S->strategy;
		r.wrap = S->wrap == B200Z_WRAP_GZIP ? B200Z_WRAP_RAW_CRC32 : S->wrap; // (gzip: the set writes header and trailer)
		r.end_mode = end_mode;
		int64_t bytes = 0;
		for (; a < due.size(); a++) {
			const int64_t b = due[a].len + (int64_t)due[a].c->history.size();
			if (!r.s.empty() && bytes + b > kSetPlanBytes) break;
			bytes += b;
			set_header(S, due[a].c);
			r.add(due[a].c, due[a].len, due[a].calls);
		}
		int rc = segments_begin(r, S->st, S->cs);
		if (r.plan) S->stats[3] = std::max(S->stats[3], b200z_plan_workspace_bytes(r.plan));
		if (!rc) rc = segments_end(r, S->st, S->cs);
		if (rc) return rc;
		S->stats[0] += (int64_t)r.s.size();
		S->stats[1]++;
	}
	return B200Z_OK;
}

// the runs a write makes due; written[i] == 0 leaves stream i out
static int set_runs(b200z_deflate_streams *S, const int32_t *op, const std::vector<char> &written) {
	const int n = (int)S->s.size();
	int rc;
	for (;;) { // (a write of more than kSetRunBytes can need more than one open run)
		std::vector<SetDue> due;
		for (int i = 0; i < n; i++) {
			SetStream *c = &S->s[(size_t)i];
			int32_t ncalls = 0;
			const int64_t avail = open_run_avail(c, S->level, &ncalls);
			if (!written[(size_t)i] || avail - c->carried < kSetRunBytes) continue;
			const int64_t len = open_run_len(c, S->level, avail, kSetRunBytes, &ncalls);
			due.push_back(SetDue{c, len, ncalls});
		}
		if (due.empty()) break;
		if ((rc = set_plans(S, B200Z_END_NONE, due))) return rc;
	}
	std::vector<SetDue> fl, fi;
	for (int i = 0; i < n; i++) {
		SetStream *c = &S->s[(size_t)i];
		if (!written[(size_t)i] || op[i] == 0) continue;
		const SetDue d{c, (int64_t)c->input.size(), (int32_t)c->chunks.size()};
		if (op[i] == 1) fl.push_back(d);
		else if (!c->flushed_once) fi.push_back(d);
		else { // Finish() right behind a Flush(): no run
			set_header(S, c);
			final_empty_block(c, S->level);
		}
	}
	if ((rc = set_plans(S, B200Z_END_FLUSH, fl)) || (rc = set_plans(S, B200Z_END_FINISH, fi))) return rc;
	for (int i = 0; i < n; i++) {
		SetStream *c = &S->s[(size_t)i];
		if (!written[(size_t)i] || op[i] == 0) continue;
		c->flushed_once = op[i] == 1;
		if (op[i] == 2) {
			stream_trailer(c, S->wrap);
			c->finished = true;
		}
	}
	return B200Z_OK;
}

// ---- Inflater handle ----------------------------------------------------------------------------------
// The reference's Inflater is a mode machine that stops at any bit and resumes (Inflater.cs:73-86, :429-552).  The kernels
// decode whole plans and report where a stream that ran out of input can be resumed (b200z_plan_get_resume_points): inside
// a Huffman block at the first symbol not decoded, otherwise at the block header it stopped in.  Between SetInput calls the
// handle keeps the window (the last 32 KiB of output), a copy of the current block's header when it stopped inside the
// block, and the compressed bytes from the resume point on; the next run enters the block through the header copy
// (b200z_inflate_plan_set_resume) and appends its output.  A stream stops inside a Huffman block only a symbol (at most 48
// bits) short of the input's end, in a header at most a header (under 600 bytes) short, and in front of a stored block at
// most 65535 + 5 bytes short: that, one header copy and the last SetInput are all the compressed bytes the handle holds,
// whatever the block size, and no byte is decoded twice.
struct InflaterH {
	bool raw = false;
	std::vector<uint8_t> input; // compressed bytes from absolute offset in_base on (what lies in front of the resume point is dropped)
	int64_t in_base = 0, in_total = 0; // in_total = bytes handed over since Reset = in_base + input.size()
	bool new_input = false;
	bool finished = false;
	bool need_dict = false;
	bool header_done = false;
	bool raw_done = false;     // the final block has ended; a zlib stream awaits its trailer at trailer_at
	int64_t trailer_at = 0;
	uint32_t read_adler = 0;   // DICTID from the header (Inflater.readAdler)
	int64_t raw_off = 0;       // where the raw deflate data starts (behind the zlib header)
	int64_t rs_bit = 0;        // resume point: bit offset from raw_off where decoding goes on -- a block header, or a symbol of
	int64_t rs_out = 0;        //   the block whose header `hdr` holds; output position there
	std::vector<uint8_t> hdr;  // that block's header bytes, from bit hdr_sbit of hdr[0] on (empty: rs_bit is a header)
	int32_t hdr_sbit = 0;
	std::vector<uint8_t> window; // last <= 32768 bytes of (dictionary ++ output[0, rs_out)): OutputWindow's contents there
	uint32_t run_adler = 1;    // Adler-32 of output[0, rs_out)
	std::vector<uint8_t> output; // decoded bytes from output position out_base on (delivered bytes in front of rs_out are dropped)
	int64_t out_base = 0;
	int64_t delivered = 0;
	int64_t consumed = 0; // bytes of input the decoder has used (header + raw + trailer), absolute
	uint32_t adler = 1;
	int error = 0;
	std::string error_msg;
	int64_t stats[4] = {0, 0, 0, 0}; // b200z_inflater_get_stats
	Staging st;
	// one plan per handle, created for capacities and run below them (b200z_inflate_plan_set_lengths): a SetInput + Inflate
	// pair costs the copies and the kernels, no allocation
	b200z_plan *plan = nullptr;
	int64_t plan_comp_cap = 0, plan_out_cap = 0;
	~InflaterH() { b200z_plan_destroy(plan); }
	int64_t out_total() const { return out_base + (int64_t)output.size(); }
	void note_held() {
		stats[2] = std::max(stats[2], (int64_t)(input.size() + hdr.size()));
		stats[3] = std::max(stats[3], (int64_t)(output.size() + window.size()));
	}
};

// checksum and window advance over the next n bytes of output, which start at output position rs_out
static int inflater_advance(InflaterH *d, int64_t n) {
	const uint8_t *seg = d->output.data() + (d->rs_out - d->out_base);
	if (!d->raw && n > 0) {
		int rc = b200z_adler32(seg, n, &d->run_adler);
		if (rc) return rc;
	}
	if (n >= 32768) d->window.assign(seg + n - 32768, seg + n);
	else {
		d->window.insert(d->window.end(), seg, seg + n);
		if (d->window.size() > 32768) d->window.erase(d->window.begin(), d->window.end() - 32768);
	}
	d->rs_out += n;
	return B200Z_OK;
}

// output in front of both the resume point and the delivery position is not needed any more.  Dropped once per run (a
// reader has usually taken everything by then): erasing it on every Inflate() would move the rest of a run's output,
// which can be 1032 times the input it came from, for every buffer handed out.
static void inflater_trim_output(InflaterH *d) {
	const int64_t keep_from = d->delivered < d->rs_out ? d->delivered : d->rs_out;
	if (keep_from > d->out_base) {
		d->output.erase(d->output.begin(), d->output.begin() + (keep_from - d->out_base));
		d->out_base = keep_from;
	}
}

// decodes from the resume point to the end of what is available; appends to output, fills consumed / raw_done and moves
// the resume point forward
static int inflater_run_device(InflaterH *d) {
	inflater_trim_output(d);
	int64_t cap = 0;
	for (int attempt = 0; attempt < 8; attempt++) {
		// slot: window image, header copy, compressed bytes from the resume point's byte on
		const int64_t tail_byte = d->rs_bit >> 3, slice_abs = d->raw_off + tail_byte;
		const int64_t avail = d->in_total - slice_abs, H = (int64_t)d->hdr.size();
		if (avail < 0 || slice_abs < d->in_base) {
			set_error("inflater resume point outside the kept input");
			return B200Z_E_INTERNAL;
		}
		const int64_t comp = H + avail, D = (int64_t)d->window.size();
		const int32_t sbit = H ? d->hdr_sbit : (int32_t)(d->rs_bit & 7);
		const int64_t skip = H ? 8 * H + (d->rs_bit & 7) : 0;
		cap = std::max(cap, comp * 8 + 65536);
		int rc;
		if (!d->plan || comp > d->plan_comp_cap || cap > d->plan_out_cap) {
			b200z_plan_destroy(d->plan);
			d->plan = nullptr;
			int64_t cc = 65536;
			while (cc < comp) cc *= 2;
			const int64_t oc = std::max(cap, cc * 8 + 65536), dc = 32768;
			if ((rc = b200z_inflate_plan_create_ex(1, &cc, &oc, B200Z_WRAP_RAW, &dc, &d->plan))) return rc;
			d->plan_comp_cap = cc;
			d->plan_out_cap = oc;
		}
		b200z_plan *plan = d->plan;
		if ((rc = b200z_inflate_plan_set_lengths(plan, &comp, &D))) return rc;
		if ((rc = b200z_inflate_plan_set_resume(plan, &sbit, &skip))) return rc;
		std::vector<uint8_t> slot;
		slot.reserve((size_t)(D + comp));
		slot.insert(slot.end(), d->window.begin(), d->window.end());
		slot.insert(slot.end(), d->hdr.begin(), d->hdr.end());
		const uint8_t *inp = d->input.data() + (slice_abs - d->in_base);
		slot.insert(slot.end(), inp, inp + avail);
		rc = handle_run(plan, d->st, slot.data(), nullptr);
		const PipeMeta &r = d->st.h;
		int64_t hb = 0, bb = 0, sb = 0, so = 0;
		if (!rc) rc = b200z_plan_get_resume_points(plan, &hb, &bb, &sb, &so, nullptr);
		if (rc) return rc;
		const int st = r.status[0] & 0xFF, detail = (r.status[0] >> 8) & 0xFF;
		const int64_t olen = r.out_len[0];
		d->stats[0]++;
		d->stats[1] += olen;
		// this run's output is output[rs_out, rs_out + olen) (what it decoded in front of an error is delivered too)
		const uint8_t *o = d->st.hout.p + plan->out_off[0];
		d->output.resize((size_t)(d->rs_out - d->out_base));
		d->output.insert(d->output.end(), o, o + olen);
		if (st != B200Z_OK && st != B200Z_E_NEED_INPUT && st != B200Z_E_NOMEM) {
			d->error = st;
			d->error_msg = inflate_detail_msg(detail);
			return B200Z_OK;
		}
		if (st == B200Z_OK) {
			d->raw_done = true;
			d->trailer_at = slice_abs + r.in_used[0] - H; // (the final block ends behind the header copy)
			d->consumed = d->trailer_at;
			return inflater_advance(d, olen);
		}
		if (so < 0 || so > olen || hb > bb || bb > sb || sb > 8 * comp || (sb < 8 * H && so != 0)) {
			set_error("inflater resume point out of range");
			return B200Z_E_INTERNAL;
		}
		if (sb >= 8 * H) { // (in front of that only when a run stopped before its first symbol)
			if ((rc = inflater_advance(d, so))) return rc;
			const uint8_t *c = slot.data() + D;
			if (bb != hb) d->hdr.assign(c + (hb >> 3), c + ((bb + 7) >> 3)); // inside a Huffman block: keep its header
			else d->hdr.clear();
			d->hdr_sbit = (int32_t)(hb & 7);
			d->rs_bit = 8 * tail_byte + (sb - 8 * H);
		}
		if (st == B200Z_E_NOMEM) {
			cap = d->plan_out_cap * 8; // (the next attempt makes a larger plan and goes on from the resume point)
			continue;
		}
		d->consumed = d->in_total;
		// compressed bytes in front of the resume point are never looked at again
		const int64_t keep_from = d->raw_off + (d->rs_bit >> 3);
		if (keep_from > d->in_base) {
			d->input.erase(d->input.begin(), d->input.begin() + (keep_from - d->in_base));
			d->in_base = keep_from;
		}
		return B200Z_OK;
	}
	set_error("output larger than any capacity tried");
	return B200Z_E_NOMEM;
}


} // namespace b200z

using namespace b200z;

extern "C" {

int b200z_deflater_create(int level, int raw, void **h) {
	if (!h) {
		set_error("h");
		return B200Z_E_ARG;
	}
	if (level == -1) level = 6;
	else if (level < 0 || level > 9) {
		set_error("level"); // ArgumentOutOfRangeException(nameof(level)), Deflater.cs:184-187
		return B200Z_E_ARG;
	}
	DeflaterH *d = new DeflaterH();
	d->level = level;
	d->raw = raw != 0;
	*h = d;
	return B200Z_OK;
}
int b200z_deflater_destroy(void *h) {
	delete (DeflaterH *)h;
	return B200Z_OK;
}
int b200z_deflater_reset(void *h) { // Deflater.Reset :204-210 keeps level and strategy
	DeflaterH *d = (DeflaterH *)h;
	d->flushing = d->finishing = d->finished = false;
	d->header_done = false;
	d->flushed_once = false;
	d->total_out = 0;
	d->dict_set = d->deflate_called = false;
	d->dict_adler = 0;
	d->draining = false;
	d->s.reset(1);
	return B200Z_OK;
}
int b200z_deflater_set_level(void *h, int level) {
	DeflaterH *d = (DeflaterH *)h;
	if (level == -1) level = 6;
	else if (level < 0 || level > 9) {
		set_error("level");
		return B200Z_E_ARG;
	}
	if (level != d->level && (!d->s.input.empty() || d->s.total_in > 0)) {
		set_error("SetLevel in mid-stream (DeflaterEngine.SetLevel flushes a block, trap T17) is not accelerated");
		return B200Z_E_UNSUPPORTED;
	}
	d->level = level;
	return B200Z_OK;
}
int b200z_deflater_get_level(void *h, int *level) {
	*level = ((DeflaterH *)h)->level;
	return B200Z_OK;
}
int b200z_deflater_set_strategy(void *h, int strategy) {
	if (strategy < 0 || strategy > 2) {
		set_error("strategy");
		return B200Z_E_ARG;
	}
	DeflaterH *d = (DeflaterH *)h;
	if (strategy != d->strategy && !d->s.input.empty()) {
		// the reference switches at the engine's current strstart (DeflaterEngine.cs:283-298), somewhere inside the input it
		// holds -- like SetLevel in mid-stream; behind a completed Flush() the switch is exact and allowed
		set_error("SetStrategy between SetInput and Flush()/Finish() is not accelerated");
		return B200Z_E_UNSUPPORTED;
	}
	d->strategy = strategy;
	return B200Z_OK;
}
int b200z_deflater_set_dictionary(void *h, const uint8_t *dict, int32_t len) {
	DeflaterH *d = (DeflaterH *)h;
	// Deflater.SetDictionary :372-381: only in INIT_STATE (before the header went out); the header's FDICT bit and
	// DICTID come from the engine's Adler-32 over the dictionary, which is then reset (:386-401)
	if (d->raw || d->deflate_called || d->header_done || d->s.total_in > 0 || d->dict_set) {
		// state != INIT_STATE (:561): a raw deflater starts in BUSY_STATE (:206), Deflate() leaves INIT_STATE (:436-464)
		set_error("SetDictionary: not in the initial state"); // InvalidOperationException
		return B200Z_E_STATE;
	}
	if (len < 0 || (len > 0 && !dict)) {
		set_error("dictionary/count");
		return B200Z_E_ARG;
	}
	uint32_t a = 1;
	if (len > 0) {
		int rc = b200z_adler32(dict, len, &a);
		if (rc) return rc;
	}
	d->dict_adler = a;
	d->dict_set = true;
	if (len < kMinMatch) return B200Z_OK; // DeflaterEngine.cs:207-210: too short to matter, not even copied
	const int32_t keep = len > kMaxDist ? kMaxDist : len; // :212-216
	carry_remember(&d->s, dict + (len - keep), (size_t)keep, 2);
	return B200Z_OK;
}
int b200z_deflater_set_input(void *h, const uint8_t *buf, int32_t len) {
	DeflaterH *d = (DeflaterH *)h;
	if (d->finishing) {
		set_error("Finish() already called"); // Deflater.cs:335
		return B200Z_E_STATE;
	}
	if (len < 0 || (len > 0 && !buf)) {
		set_error("buffer/count");
		return B200Z_E_ARG;
	}
	// (no length limit: Deflate() runs long input in open runs, so a closing run holds at most what the last one carried,
	// kOpenRunBytes and one SetInput of at most 2^31 - 1 bytes, and plans take a stream position of any size)
	if (len > 0) d->flushed_once = false;
	d->s.input.insert(d->s.input.end(), buf, buf + len);
	if (len > 0) {
		// engine.NeedsInput (DeflaterEngine.cs:187-190) is false until Deflate() has taken the bytes; a zero-length SetInput
		// leaves it true, so the stream classes do not even call Deflate() for it
		d->s.undrained = true;
		if (d->level <= 4) d->s.chunks.push_back(len); // the schedule matters for DeflateStored / DeflateFast only (trap T9)
	}
	return B200Z_OK;
}
int b200z_deflater_flush(void *h) {
	((DeflaterH *)h)->flushing = true;
	return B200Z_OK;
}
int b200z_deflater_finish(void *h) {
	DeflaterH *d = (DeflaterH *)h;
	d->flushing = d->finishing = true;
	return B200Z_OK;
}

int b200z_deflater_deflate(void *h, uint8_t *out, int32_t cap, int32_t *produced) {
	DeflaterH *d = (DeflaterH *)h;
	if (!produced || cap < 0 || (cap > 0 && !out)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	*produced = 0;
	d->deflate_called = true;
	if (!d->flushing && !d->finishing) d->s.undrained = false; // BUSY_STATE: the engine takes everything SetInput handed over
	if (!d->finished) { // (also in front of a Flush() / Finish() run: no run sees more than one run's worth of new input)
		int rc = deflater_open_runs(d);
		if (rc) return rc;
	}
	// make output due (Deflater.Deflate :427-522)
	if (!d->finished && d->s.pending_pos == d->s.pending.size() && (d->flushing || d->finishing)) {
		d->s.pending.clear();
		d->s.pending_pos = 0;
		deflater_header(d);
		if (d->finishing) {
			if (d->flushed_once) {
				final_empty_block(&d->s, d->level);
			} else {
				int rc = deflater_run_device(d, B200Z_END_FINISH, (int64_t)d->s.input.size(), (int32_t)d->s.chunks.size());
				if (rc) return rc;
			}
			stream_trailer(&d->s, d->raw ? B200Z_WRAP_RAW : B200Z_WRAP_ZLIB);
			d->finished = true;
		} else {
			// sync flush (level 0 skips the padding, :488)
			int rc = deflater_run_device(d, B200Z_END_FLUSH, (int64_t)d->s.input.size(), (int32_t)d->s.chunks.size());
			if (rc) return rc;
			d->flushed_once = true;
			d->flushing = false;
		}
	}
	size_t avail = d->s.pending.size() - d->s.pending_pos;
	size_t take = avail < (size_t)cap ? avail : (size_t)cap;
	if (take) memcpy(out, d->s.pending.data() + d->s.pending_pos, take);
	d->s.pending_pos += take;
	d->total_out += (int64_t)take;
	*produced = (int32_t)take;
	if (d->s.pending_pos == d->s.pending.size()) d->draining = false;
	return B200Z_OK;
}
int b200z_deflater_needs_input(void *h, int *flag) {
	// DeflaterEngine.NeedsInput (:187-190): false between SetInput and the Deflate() call that takes the bytes.  The
	// handle copies on SetInput, but it reports what the reference reports: DeflaterOutputStream.Write calls Deflate()
	// exactly while this is false (Streams/DeflaterOutputStream.cs:245-275), and whether that call happened before
	// Flush() / Finish() changes the bytes at levels 0-4 (b200z_history.undrained_last).  The output of an open run also
	// keeps it false until it has been handed out, as the reference's engine holds input while its output is pending.
	const DeflaterH *d = (const DeflaterH *)h;
	*flag = (d->s.undrained || d->draining) ? 0 : 1;
	return B200Z_OK;
}
int b200z_deflater_is_finished(void *h, int *flag) {
	DeflaterH *d = (DeflaterH *)h;
	*flag = (d->finished && d->s.pending_pos == d->s.pending.size()) ? 1 : 0; // Deflater.cs:271-277
	return B200Z_OK;
}
int b200z_deflater_total_in(void *h, int64_t *v) {
	DeflaterH *d = (DeflaterH *)h;
	*v = d->s.total_in;
	return B200Z_OK;
}
int b200z_deflater_total_out(void *h, int64_t *v) {
	*v = ((DeflaterH *)h)->total_out;
	return B200Z_OK;
}
int b200z_deflater_adler(void *h, uint32_t *v) {
	DeflaterH *d = (DeflaterH *)h;
	*v = d->raw ? 0u : d->s.check;
	return B200Z_OK;
}

int b200z_inflater_create(int raw, void **h) {
	if (!h) {
		set_error("h");
		return B200Z_E_ARG;
	}
	InflaterH *d = new InflaterH();
	d->raw = raw != 0;
	*h = d;
	return B200Z_OK;
}
int b200z_inflater_destroy(void *h) {
	delete (InflaterH *)h;
	return B200Z_OK;
}
int b200z_inflater_reset(void *h) {
	InflaterH *d = (InflaterH *)h;
	d->input.clear();
	d->output.clear();
	d->window.clear();
	d->new_input = d->finished = d->need_dict = d->header_done = d->raw_done = false;
	d->in_base = d->in_total = 0;
	d->trailer_at = 0;
	d->raw_off = 0;
	d->rs_bit = d->rs_out = 0;
	d->hdr.clear();
	d->hdr_sbit = 0;
	for (int64_t &v : d->stats) v = 0;
	d->run_adler = 1;
	d->out_base = 0;
	d->delivered = 0;
	d->consumed = 0;
	d->adler = 1;
	d->error = 0;
	d->read_adler = 0;
	return B200Z_OK;
}
int b200z_inflater_set_dictionary(void *h, const uint8_t *dict, int32_t len) {
	InflaterH *d = (InflaterH *)h;
	// Inflater.SetDictionary :589-620
	if (len < 0 || (len > 0 && !dict)) {
		set_error("buffer/count");
		return B200Z_E_ARG;
	}
	if (!d->need_dict) {
		set_error("Dictionary is not needed"); // InvalidOperationException
		return B200Z_E_STATE;
	}
	uint32_t a = 1;
	if (len > 0) {
		int rc = b200z_adler32(dict, len, &a);
		if (rc) return rc;
	}
	if (a != d->read_adler) {
		set_error("Wrong adler checksum"); // SharpZipBaseException
		return B200Z_E_DATA;
	}
	const int32_t keep = len > 32768 ? 32768 : len; // OutputWindow.CopyDict :160-166
	d->window.assign(dict + (len - keep), dict + len);
	d->need_dict = false;
	d->adler = 1;
	d->new_input = true; // what was handed over behind the header can be decoded now
	return B200Z_OK;
}
int b200z_inflater_set_input(void *h, const uint8_t *buf, int32_t len) {
	InflaterH *d = (InflaterH *)h;
	if (len < 0 || (len > 0 && !buf)) {
		set_error("buffer/count");
		return B200Z_E_ARG;
	}
	if (d->in_total > d->consumed && !d->finished) {
		set_error("Old input was not completely processed"); // StreamManipulator.cs:263
		return B200Z_E_STATE;
	}
	if (d->finished) {
		// after the end of the stream the reference keeps unread bytes as RemainingInput; replace them
		d->input.resize((size_t)(d->consumed - d->in_base));
		d->in_total = d->consumed;
	}
	d->input.insert(d->input.end(), buf, buf + len);
	d->in_total += len;
	d->new_input = true;
	d->note_held();
	return B200Z_OK;
}

int b200z_inflater_inflate(void *h, uint8_t *out, int32_t cap, int32_t *produced) {
	InflaterH *d = (InflaterH *)h;
	if (!produced || cap < 0 || (cap > 0 && !out)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	*produced = 0;
	if (d->error) {
		set_error("%s", d->error_msg.c_str());
		return d->error;
	}
	if (!d->finished && d->new_input) {
		d->new_input = false;
		if (!d->raw && !d->header_done) {
			// (nothing is dropped from `input` before the header is done: in_base == 0 here)
			if (d->input.size() < 2) {
				d->consumed = (int64_t)d->input.size();
				return B200Z_OK; // DecodeHeader needs 16 bits (Inflater.cs:209-215)
			}
			const int header = (d->input[0] << 8) | d->input[1];
			if (header % 31 != 0) {
				d->error = B200Z_E_DATA;
				d->error_msg = "Header checksum illegal";
			} else if ((header & 0x0f00) != (8 << 8)) {
				d->error = B200Z_E_DATA;
				d->error_msg = "Compression Method unknown";
			}
			if (d->error) {
				set_error("%s", d->error_msg.c_str());
				return d->error;
			}
			if (header & 0x0020) {
				// PRESET_DICT: DecodeDict reads the 4-byte DICTID MSB first (:185-203); Inflate() then returns 0 until
				// SetDictionary supplies a dictionary with that Adler-32
				if (d->input.size() < 6) {
					d->consumed = (int64_t)d->input.size();
					return B200Z_OK;
				}
				d->read_adler = ((uint32_t)d->input[2] << 24) | ((uint32_t)d->input[3] << 16) | ((uint32_t)d->input[4] << 8) | d->input[5];
				d->need_dict = true;
				d->adler = d->read_adler; // Inflater.Adler reports readAdler while the dictionary is awaited (:823-836)
				d->header_done = true;
				d->raw_off = 6;
				d->consumed = 6;
				d->new_input = true; // the bytes behind the DICTID wait for SetDictionary
				return B200Z_OK;
			}
			d->header_done = true;
			d->raw_off = 2;
		}
		if (d->need_dict) {
			d->new_input = true;
			return B200Z_OK;
		}
		if (!d->raw_done) {
			int rc = inflater_run_device(d);
			d->note_held();
			if (rc) return rc;
		}
		if (d->raw_done && d->raw) {
			d->finished = true;
		} else if (d->raw_done) {
			// Adler32 trailer, read MSB first (DecodeChksum :397-418); until it is complete only its bytes are awaited, the
			// decoded output is all there
			if (d->in_total - d->trailer_at < 4) {
				d->consumed = d->in_total;
			} else {
				const uint8_t *t = d->input.data() + (d->trailer_at - d->in_base);
				const uint32_t want = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
				d->adler = d->run_adler; // of all the output
				if (d->run_adler != want) {
					d->error = B200Z_E_DATA;
					d->error_msg = "Adler chksum doesn't match";
				}
				d->consumed = d->trailer_at + 4;
				d->finished = true;
			}
		}
	}
	size_t avail = (size_t)(d->out_total() - d->delivered);
	size_t take = avail < (size_t)cap ? avail : (size_t)cap;
	if (take) memcpy(out, d->output.data() + (d->delivered - d->out_base), take);
	d->delivered += (int64_t)take;
	*produced = (int32_t)take;
	if (take == 0 && d->error) {
		set_error("%s", d->error_msg.c_str());
		return d->error;
	}
	return B200Z_OK;
}
int b200z_inflater_needs_input(void *h, int *flag) {
	InflaterH *d = (InflaterH *)h;
	*flag = (d->in_total <= d->consumed) ? 1 : 0; // StreamManipulator.IsNeedingInput
	return B200Z_OK;
}
int b200z_inflater_needs_dictionary(void *h, int *flag) {
	*flag = ((InflaterH *)h)->need_dict ? 1 : 0; // mode == DECODE_DICT && neededBits == 0 (Inflater.cs:792-798)
	return B200Z_OK;
}
int b200z_inflater_is_finished(void *h, int *flag) {
	InflaterH *d = (InflaterH *)h;
	// Inflater.cs:806-812; a trailer that did not verify is an exception from Inflate() in the reference (DecodeChksum
	// :397-418), so the stream is not "finished" as long as that error has not been delivered
	*flag = (d->finished && !d->error && d->delivered == d->out_total()) ? 1 : 0;
	return B200Z_OK;
}
int b200z_inflater_remaining_input(void *h, int32_t *v) {
	InflaterH *d = (InflaterH *)h;
	*v = (int32_t)(d->in_total - d->consumed);
	return B200Z_OK;
}
int b200z_inflater_total_in(void *h, int64_t *v) {
	*v = ((InflaterH *)h)->consumed; // totalIn - RemainingInput (Inflater.cs:862-868)
	return B200Z_OK;
}
int b200z_inflater_total_out(void *h, int64_t *v) {
	*v = ((InflaterH *)h)->delivered;
	return B200Z_OK;
}
int b200z_inflater_adler(void *h, uint32_t *v) {
	InflaterH *d = (InflaterH *)h;
	*v = d->raw ? 0u : d->adler;
	return B200Z_OK;
}
int b200z_inflater_get_stats(void *h, int64_t *v, int32_t cap) {
	if (!h || cap < 0 || (cap > 0 && !v)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const InflaterH *d = (const InflaterH *)h;
	for (int32_t i = 0; i < cap && i < 4; i++) v[i] = d->stats[i];
	return B200Z_OK;
}

int b200z_deflate_streams_create(int32_t n, int level, int strategy, int wrap, b200z_deflate_streams **s) {
	if (!s || n < 0) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (level == -1) level = 6;
	if (level < 0 || level > 9 || strategy < 0 || strategy > 2 || wrap < B200Z_WRAP_RAW || wrap > B200Z_WRAP_RAW_CRC32) {
		set_error("level/strategy/wrap");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	b200z_deflate_streams *S = new b200z_deflate_streams();
	S->device = current_device();
	DeviceGuard guard(S->device);
	S->level = level;
	S->strategy = strategy;
	S->wrap = wrap;
	S->s = std::vector<SetStream>((size_t)n);
	for (SetStream &c : S->s) c.check = wrap == B200Z_WRAP_ZLIB ? 1u : 0u; // Adler32.Reset / Crc32.Reset
	if (cudaStreamCreateWithFlags(&S->cs, cudaStreamNonBlocking) != cudaSuccess) {
		delete S;
		set_error("cudaStreamCreate failed");
		return B200Z_E_CUDA;
	}
	*s = S;
	return B200Z_OK;
}

int b200z_deflate_streams_write(b200z_deflate_streams *S, const uint8_t *const *in, const int64_t *len, const int32_t *op, int32_t *status) {
	if (!S || (!S->s.empty() && (!in || !len || !op || !status))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const int n = (int)S->s.size();
	for (int i = 0; i < n; i++) // (nothing is taken when an argument is bad)
		if (len[i] < 0 || (len[i] > 0 && !in[i]) || op[i] < 0 || op[i] > 2) {
			set_error("stream %d: buffer/count/op", i);
			return B200Z_E_ARG;
		}
	if (S->broken) {
		set_error("an earlier run of this Deflater set failed with status %d", S->broken);
		return S->broken;
	}
	DeviceGuard guard(S->device);
	int first = -1;
	std::vector<char> written((size_t)n, 0);
	for (int i = 0; i < n; i++) {
		SetStream &c = S->s[(size_t)i];
		status[i] = B200Z_OK;
		if (c.finished) { // Deflater.SetInput: "Finish() already called" (Deflater.cs:335); nothing at all is no call
			if (len[i] > 0 || op[i] != 0) {
				status[i] = B200Z_E_STATE;
				if (first < 0) first = i;
			}
			continue;
		}
		written[(size_t)i] = 1;
		c.input.insert(c.input.end(), in[i], in[i] + len[i]);
		if (len[i] > 0) {
			c.flushed_once = false;
			if (S->level <= 4) c.chunks.push_back(len[i]); // the schedule (trap T9); every write drains, so none is undrained
		}
		S->stats[2] = std::max(S->stats[2], (int64_t)c.input.size());
	}
	const int rc = set_runs(S, op, written);
	if (rc) {
		S->broken = rc;
		return rc;
	}
	if (first >= 0) {
		set_error("stream %d: Finish() already called", first);
		return B200Z_E_STATE;
	}
	return B200Z_OK;
}

int b200z_deflate_streams_read(b200z_deflate_streams *S, uint8_t *const *out, const int64_t *cap, int64_t *got) {
	if (!S || (!S->s.empty() && (!out || !cap || !got))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const int n = (int)S->s.size();
	for (int i = 0; i < n; i++)
		if (cap[i] < 0 || (cap[i] > 0 && !out[i])) {
			set_error("stream %d: buffer/count", i);
			return B200Z_E_ARG;
		}
	for (int i = 0; i < n; i++) {
		SetStream &c = S->s[(size_t)i];
		const int64_t take = std::min<int64_t>(cap[i], (int64_t)(c.pending.size() - c.pending_pos));
		if (take > 0) memcpy(out[i], c.pending.data() + c.pending_pos, (size_t)take);
		c.pending_pos += (size_t)take;
		got[i] = take;
		if (c.pending_pos == c.pending.size()) {
			c.pending.clear();
			c.pending_pos = 0;
		}
	}
	return B200Z_OK;
}

int b200z_deflate_streams_check(b200z_deflate_streams *S, uint32_t *check) {
	if (!S || (!S->s.empty() && !check)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	for (size_t i = 0; i < S->s.size(); i++) check[i] = S->wrap == B200Z_WRAP_RAW ? 0u : S->s[i].check;
	return B200Z_OK;
}

int b200z_deflate_streams_stats(b200z_deflate_streams *S, int64_t *v, int32_t cap) {
	if (!S || cap < 0 || (cap > 0 && !v)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	for (int32_t i = 0; i < cap && i < 4; i++) v[i] = S->stats[i];
	return B200Z_OK;
}

int b200z_deflate_streams_destroy(b200z_deflate_streams *S) {
	if (!S) return B200Z_OK;
	DeviceGuard guard(S->device); // (the device buffers go while the set's device is current)
	if (S->cs) {
		cudaStreamSynchronize(S->cs);
		cudaStreamDestroy(S->cs);
	}
	delete S;
	return B200Z_OK;
}

} // extern "C"
