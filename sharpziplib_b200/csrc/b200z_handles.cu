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

// ---- Inflater streams: the Inflater handle and the Inflater set share one host path ---------------------------------
// The reference's Inflater is a mode machine that stops at any bit and resumes (Inflater.cs:73-86, :429-552).  The kernels
// decode whole plans and report where a stream that ran out of input can be resumed (b200z_plan_get_resume_points): inside
// a Huffman block at the first symbol not decoded, otherwise at the block header it stopped in.  Between runs a stream
// keeps its window (the last 32 KiB of output) in a device window pool, a copy of the current block's header when it
// stopped inside the block, and the compressed bytes from the resume point on; the next run enters the block through the
// header copy (b200z_inflate_plan_set_resume) and appends its output.  A stream stops inside a Huffman block only a symbol
// (at most 48 bits) short of the input's end, in a header at most a header (under 600 bytes) short, and in front of a
// stored block at most 65535 + 5 bytes short: that, one header copy and the last SetInput are all the compressed bytes a
// stream holds, whatever the block size, and no byte is decoded twice.

// What one Inflater stream carries between device runs, whoever drives it (a handle, or a stream of a set).
struct InflateCarry {
	int wrap = B200Z_WRAP_RAW; // RAW, ZLIB (Adler-32 and the zlib framing) or RAW_CRC32 (a CRC-32)
	int32_t pool = 0;          // the stream's slot in its owner's window pool
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
	int32_t win_len = 0;       // last <= 32768 bytes of (dictionary ++ output[0, rs_out)), in the pool slot
	uint32_t run_check = 1;    // Adler-32 / CRC-32 of output[0, rs_out)
	std::vector<uint8_t> output; // decoded bytes from output position out_base on (delivered bytes in front of rs_out are dropped)
	int64_t out_base = 0;
	int64_t delivered = 0;
	int64_t consumed = 0; // bytes of input the decoder has used (header + raw + trailer), absolute
	uint32_t adler = 1;   // what Inflater.Adler reports (the handle)
	int32_t error = 0;    // code | detail << 8 of the stream's data error
	int64_t out_need = 0; // B200Z_E_NOMEM: the output capacity the next run asks for
	int attempts = 0;     // runs in a row that ended in B200Z_E_NOMEM
	int64_t decoded = 0;  // output bytes the runs produced (bytes decoded twice counted twice)
	int64_t max_comp = 0, max_out = 0; // the most compressed / output bytes held at once
	int64_t out_total() const { return out_base + (int64_t)output.size(); }
	int ck_kind() const { return wrap == B200Z_WRAP_ZLIB ? 1 : (wrap == B200Z_WRAP_RAW_CRC32 ? 0 : -1); }
	void note_held() {
		max_comp = std::max(max_comp, (int64_t)(input.size() + hdr.size()));
		max_out = std::max(max_out, (int64_t)output.size() + win_len);
	}
	void reset() { // (keeps wrap and pool)
		const int w = wrap;
		const int32_t p = pool;
		*this = InflateCarry();
		wrap = w;
		pool = p;
		run_check = w == B200Z_WRAP_RAW_CRC32 ? 0u : 1u; // Crc32.Reset / Adler32.Reset
	}
};

// What the runs of one owner (a handle, a set) share on the device: the window pool, the packed upload and the slot
// descriptors, the staging of its plans, and what it counts.
struct CarryDevice {
	DevBuf pool, packed, slots;
	Staging st;
	int64_t h2d = 0;                     // host-to-device bytes the runs copied
	int64_t plans_created = 0, workspace = 0;
	int ensure_pool(int32_t n) { return pool.ensure((size_t)std::max<int32_t>(n, 1) * (size_t)kCarryWindow); }
};

// A raw inflate plan kept between runs, with the capacities it was created for (b200z_inflate_plan_set_lengths runs it
// below them).
struct CarryPlan {
	b200z_plan *plan = nullptr;
	std::vector<int64_t> comp_cap, out_cap;
	CarryPlan() = default;
	CarryPlan(CarryPlan &&o) noexcept : plan(o.plan), comp_cap(std::move(o.comp_cap)), out_cap(std::move(o.out_cap)) { o.plan = nullptr; }
	CarryPlan(const CarryPlan &) = delete;
	~CarryPlan() { b200z_plan_destroy(plan); }
};

// A run's compressed capacity: a power of two with room for the header copy and the bytes kept in front of a resume
// point, so that equal pieces fit the plan their first run made.
static int64_t carry_comp_cap(int64_t comp) {
	int64_t cc = 65536;
	while (cc < comp + 1024) cc *= 2;
	return cc;
}
static int64_t carry_out_need(const InflateCarry *c, int64_t comp) { return std::max(c->out_need, comp * 8 + 65536); }

// output in front of both the resume point and the delivery position is not needed any more.  Dropped once per run (a
// reader has usually taken everything by then): erasing it on every Inflate() would move the rest of a run's output,
// which can be 1032 times the input it came from, for every buffer handed out.
static void carry_trim_output(InflateCarry *c) {
	const int64_t keep_from = c->delivered < c->rs_out ? c->delivered : c->rs_out;
	if (keep_from > c->out_base) {
		c->output.erase(c->output.begin(), c->output.begin() + (keep_from - c->out_base));
		c->out_base = keep_from;
	}
}

// The compressed bytes of a stream's next run: the header copy, then the input from the resume point's byte on.
struct CarryCut {
	int64_t tail_byte, slice_abs, avail, H, comp;
};
static CarryCut carry_cut(const InflateCarry *c) {
	CarryCut u;
	u.tail_byte = c->rs_bit >> 3;
	u.slice_abs = c->raw_off + u.tail_byte;
	u.avail = c->in_total - u.slice_abs;
	u.H = (int64_t)c->hdr.size();
	u.comp = u.H + u.avail;
	return u;
}

// One device run of k streams as one raw inflate plan, on `cs`: each stream decodes from its resume point to the end of
// what it holds, appends to its output, fills consumed / raw_done, and moves its resume point, window and running
// checksum forward.  The run synchronises `cs` twice: once for the statuses and resume points, once for the output bytes
// and checksums.  A stream whose output outgrew its capacity (B200Z_E_NOMEM) goes on from its resume point: it comes back
// with out_need set for a later run.  A stream with corrupt data gets its error; the bytes in front of it are delivered.
static int inflate_run(CarryDevice &dv, CarryPlan &cp, const std::vector<InflateCarry *> &s, cudaStream_t cs) {
	const int k = (int)s.size();
	std::vector<CarryCut> cut((size_t)k);
	std::vector<int64_t> comp((size_t)k), D((size_t)k), skip((size_t)k), need((size_t)k);
	std::vector<int32_t> sbit((size_t)k);
	bool fits = cp.plan && cp.plan->n == k;
	for (int i = 0; i < k; i++) {
		InflateCarry *c = s[(size_t)i];
		carry_trim_output(c);
		const CarryCut &u = cut[(size_t)i] = carry_cut(c);
		if (u.avail < 0 || u.slice_abs < c->in_base) {
			set_error("inflater resume point outside the kept input");
			return B200Z_E_INTERNAL;
		}
		comp[(size_t)i] = u.comp;
		D[(size_t)i] = c->win_len;
		sbit[(size_t)i] = u.H ? c->hdr_sbit : (int32_t)(c->rs_bit & 7);
		skip[(size_t)i] = u.H ? 8 * u.H + (c->rs_bit & 7) : 0;
		need[(size_t)i] = carry_out_need(c, u.comp);
		if (fits && (u.comp > cp.comp_cap[(size_t)i] || need[(size_t)i] > cp.out_cap[(size_t)i])) fits = false;
	}
	int rc;
	if (!fits) {
		b200z_plan_destroy(cp.plan);
		cp.plan = nullptr;
		cp.comp_cap.resize((size_t)k);
		cp.out_cap.resize((size_t)k);
		for (int i = 0; i < k; i++) {
			cp.comp_cap[(size_t)i] = carry_comp_cap(comp[(size_t)i]);
			cp.out_cap[(size_t)i] = std::max(need[(size_t)i], cp.comp_cap[(size_t)i] * 8 + 65536);
		}
		const std::vector<int64_t> dc((size_t)k, kCarryWindow);
		if ((rc = b200z_inflate_plan_create_ex(k, cp.comp_cap.data(), cp.out_cap.data(), B200Z_WRAP_RAW, dc.data(), &cp.plan))) return rc;
		dv.plans_created++;
		dv.workspace = std::max(dv.workspace, b200z_plan_workspace_bytes(cp.plan));
	}
	b200z_plan *plan = cp.plan;
	if ((rc = b200z_inflate_plan_set_lengths(plan, comp.data(), D.data()))) return rc;
	if ((rc = b200z_inflate_plan_set_resume(plan, sbit.data(), skip.data()))) return rc;
	dv.h2d += 24ll * k; // (the lengths, start bits and jumps the two calls above write into the plan's workspace)
	if ((rc = dv.st.ensure(plan, false))) return rc;
	Staging &st = dv.st;
	// one packed upload of every stream's header copy and compressed bytes; k_carry_stage puts them and the pool's windows
	// into the slots
	std::vector<CarrySlot> slot((size_t)k);
	int64_t pk = 0;
	for (int i = 0; i < k; i++) {
		const InflateCarry *c = s[(size_t)i];
		const CarryCut &u = cut[(size_t)i];
		CarrySlot &sl = slot[(size_t)i];
		sl.pk_off = pk;
		sl.data_off = b200z_plan_data_offset(plan, i);
		sl.comp = u.comp;
		sl.out_off = plan->out_off[(size_t)i];
		sl.out_pos = 0;
		sl.pool = c->pool;
		sl.win_len = c->win_len;
		if (u.H) memcpy(st.hin.p + pk, c->hdr.data(), (size_t)u.H);
		if (u.avail) memcpy(st.hin.p + pk + u.H, c->input.data() + (u.slice_abs - c->in_base), (size_t)u.avail);
		pk = align_up(pk + u.comp, 16);
	}
	const size_t slot_bytes = sizeof(CarrySlot) * (size_t)k;
	if ((rc = dv.packed.ensure((size_t)pk + 16)) || (rc = dv.slots.ensure(slot_bytes))) return rc;
	if (pk) B200Z_CUDA(cudaMemcpyAsync(dv.packed.p, st.hin.p, (size_t)pk, cudaMemcpyHostToDevice, cs));
	B200Z_CUDA(cudaMemcpyAsync(dv.slots.p, slot.data(), slot_bytes, cudaMemcpyHostToDevice, cs));
	dv.h2d += pk + (int64_t)slot_bytes;
	const CarrySlot *d_slots = reinterpret_cast<const CarrySlot *>(dv.slots.p);
	if ((rc = carry_stage_launch(d_slots, k, dv.pool.p, dv.packed.p, st.din.p, cs))) return rc;
	if ((rc = b200z_plan_run(plan, st.din.p, st.dout.p, st.d.out_len, st.d.status, st.d.check, st.d.in_used, cs))) return rc;
	B200Z_CUDA(cudaMemcpyAsync(st.h.out_len, st.d.out_len, (size_t)k * (8 + 8 + 4 + 4), cudaMemcpyDeviceToHost, cs));
	std::vector<int64_t> hb((size_t)k), bb((size_t)k), sb((size_t)k), so((size_t)k);
	if ((rc = b200z_plan_get_resume_points(plan, hb.data(), bb.data(), sb.data(), so.data(), cs))) return rc; // (synchronises cs)
	const PipeMeta &m = st.h;
	// how far each stream's window and checksum move: all of a finished stream's output, up to the resume point otherwise
	std::vector<int64_t> adv((size_t)k, 0), ck_off((size_t)k);
	for (int i = 0; i < k; i++) {
		const int code = m.status[i] & 0xFF;
		const int64_t olen = m.out_len[i], H = cut[(size_t)i].H;
		const int64_t sbi = sb[(size_t)i], soi = so[(size_t)i];
		if (code == B200Z_OK) adv[(size_t)i] = olen;
		else if (code == B200Z_E_NEED_INPUT || code == B200Z_E_NOMEM) {
			if (soi < 0 || soi > olen || hb[(size_t)i] > bb[(size_t)i] || bb[(size_t)i] > sbi || sbi > 8 * comp[(size_t)i] || (sbi < 8 * H && soi != 0)) {
				set_error("inflater resume point out of range");
				return B200Z_E_INTERNAL;
			}
			if (sbi >= 8 * H) adv[(size_t)i] = soi; // (in front of that only when a run stopped before its first symbol)
		}
		slot[(size_t)i].out_pos = adv[(size_t)i];
		ck_off[(size_t)i] = plan->out_off[(size_t)i];
	}
	B200Z_CUDA(cudaMemcpyAsync(dv.slots.p, slot.data(), slot_bytes, cudaMemcpyHostToDevice, cs));
	dv.h2d += (int64_t)slot_bytes;
	if ((rc = carry_window_launch(d_slots, k, st.din.p, st.dout.p, dv.pool.p, cs))) return rc;
	for (int i = 0; i < k; i++)
		if (m.out_len[i] > 0)
			B200Z_CUDA(cudaMemcpyAsync(st.hout.p + plan->out_off[(size_t)i], st.dout.p + plan->out_off[(size_t)i], (size_t)m.out_len[i],
			                           cudaMemcpyDeviceToHost, cs));
	// the running checksums go on over the output the run left on the device; seeds and results live in the pinned
	// metadata, which the device reads and writes in place (pinned memory is mapped under unified addressing)
	const int kind = s[0]->ck_kind();
	if (kind >= 0) {
		for (int i = 0; i < k; i++) m.check[i] = s[(size_t)i]->run_check;
		rc = b200z_checksum_batch_device(kind, st.dout.p, ck_off.data(), adv.data(), k, m.check, cs); // (synchronises cs)
		dv.h2d += 16ll * k;
		if (rc) return rc;
	} else {
		B200Z_CUDA(cudaStreamSynchronize(cs));
	}
	for (int i = 0; i < k; i++) {
		InflateCarry *c = s[(size_t)i];
		const CarryCut &u = cut[(size_t)i];
		const int code = m.status[i] & 0xFF;
		const int64_t olen = m.out_len[i];
		// this run's output is output[rs_out, rs_out + olen) (what it decoded in front of an error is delivered too)
		const uint8_t *o = st.hout.p + plan->out_off[(size_t)i];
		c->output.resize((size_t)(c->rs_out - c->out_base));
		c->output.insert(c->output.end(), o, o + olen);
		c->decoded += olen;
		c->out_need = 0;
		if (code != B200Z_OK && code != B200Z_E_NEED_INPUT && code != B200Z_E_NOMEM) {
			c->error = m.status[i];
			c->attempts = 0;
			continue;
		}
		const int64_t a = adv[(size_t)i];
		if (kind >= 0) c->run_check = m.check[i];
		c->win_len = (int32_t)std::min<int64_t>(kCarryWindow, c->win_len + a);
		c->rs_out += a;
		if (code == B200Z_OK) {
			c->raw_done = true;
			c->trailer_at = u.slice_abs + m.in_used[i] - u.H; // (the final block ends behind the header copy)
			c->consumed = c->trailer_at;
			c->attempts = 0;
			continue;
		}
		const int64_t sbi = sb[(size_t)i];
		if (sbi >= 8 * u.H) {
			const uint8_t *p = st.hin.p + slot[(size_t)i].pk_off; // (the header copy, then the compressed bytes)
			if (bb[(size_t)i] != hb[(size_t)i]) c->hdr.assign(p + (hb[(size_t)i] >> 3), p + ((bb[(size_t)i] + 7) >> 3)); // inside a Huffman block: keep its header
			else c->hdr.clear();
			c->hdr_sbit = (int32_t)(hb[(size_t)i] & 7);
			c->rs_bit = 8 * u.tail_byte + (sbi - 8 * u.H);
		}
		if (code == B200Z_E_NOMEM) {
			c->out_need = cp.out_cap[(size_t)i] * 8; // (the next run makes a larger plan and goes on from the resume point)
			c->attempts++;
			continue;
		}
		c->attempts = 0;
		c->consumed = c->in_total;
		// compressed bytes in front of the resume point are never looked at again
		const int64_t keep_from = c->raw_off + (c->rs_bit >> 3);
		if (keep_from > c->in_base) {
			c->input.erase(c->input.begin(), c->input.begin() + (keep_from - c->in_base));
			c->in_base = keep_from;
		}
	}
	return B200Z_OK;
}

// A run takes a stream that has input it has not decoded, its zlib header read, no dictionary awaited, no error and
// its final block not yet ended.  Only a stream whose last run ran out of output capacity goes on without new input.
static bool carry_runs(const InflateCarry *c) { return !c->error && !c->need_dict && !c->raw_done && !c->finished; }

// zlib: reads the header (Inflater.DecodeHeader :209-255) and the DICTID (DecodeDict :185-203) once their bytes are
// there.  False while they are not, on an error and while a preset dictionary is awaited: the stream does not run.
static bool carry_header(InflateCarry *c) {
	if (c->wrap == B200Z_WRAP_ZLIB && !c->header_done) {
		// (nothing is dropped from `input` before the header is done: in_base == 0 here)
		if (c->input.size() < 2) {
			c->consumed = (int64_t)c->input.size();
			return false; // DecodeHeader needs 16 bits (Inflater.cs:209-215)
		}
		const int header = (c->input[0] << 8) | c->input[1];
		if (header % 31 != 0) c->error = B200Z_E_DATA | 19 << 8;            // "Header checksum illegal"
		else if ((header & 0x0f00) != (8 << 8)) c->error = B200Z_E_DATA | 20 << 8; // "Compression Method unknown"
		if (c->error) return false;
		if (header & 0x0020) {
			// PRESET_DICT: DecodeDict reads the 4-byte DICTID MSB first (:185-203); Inflate() then returns 0 until
			// SetDictionary supplies a dictionary with that Adler-32
			if (c->input.size() < 6) {
				c->consumed = (int64_t)c->input.size();
				return false;
			}
			c->read_adler = ((uint32_t)c->input[2] << 24) | ((uint32_t)c->input[3] << 16) | ((uint32_t)c->input[4] << 8) | c->input[5];
			c->need_dict = true;
			c->adler = c->read_adler; // Inflater.Adler reports readAdler while the dictionary is awaited (:823-836)
			c->header_done = true;
			c->raw_off = 6;
			c->consumed = 6;
			c->new_input = true; // the bytes behind the DICTID wait for SetDictionary
			return false;
		}
		c->header_done = true;
		c->raw_off = 2;
	}
	if (c->need_dict) {
		c->new_input = true;
		return false;
	}
	return true;
}

// behind the final block: a zlib stream's Adler-32 trailer, read MSB first (DecodeChksum :397-418); until it is complete
// only its bytes are awaited, the decoded output is all there
static void carry_trailer(InflateCarry *c) {
	if (!c->raw_done || c->finished) return;
	if (c->wrap != B200Z_WRAP_ZLIB) {
		c->finished = true;
		return;
	}
	if (c->in_total - c->trailer_at < 4) {
		c->consumed = c->in_total;
		return;
	}
	const uint8_t *t = c->input.data() + (c->trailer_at - c->in_base);
	const uint32_t want = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
	c->adler = c->run_check; // of all the output
	if (c->run_check != want) c->error = B200Z_E_DATA | 11 << 8; // "Adler chksum doesn't match"
	c->consumed = c->trailer_at + 4;
	c->finished = true;
}

// SetInput (the reference copies nothing; the carry keeps the bytes until they are decoded)
static void carry_input(InflateCarry *c, const uint8_t *buf, int64_t len) {
	if (c->finished) {
		// after the end of the stream the reference keeps unread bytes as RemainingInput; replace them
		c->input.resize((size_t)(c->consumed - c->in_base));
		c->in_total = c->consumed;
	}
	c->input.insert(c->input.end(), buf, buf + len);
	c->in_total += len;
	c->new_input = true;
	c->note_held();
}

// Inflater.SetDictionary :589-620: the dictionary's tail becomes the window in the stream's pool slot, the one time a
// window crosses PCIe
static int carry_set_dictionary(CarryDevice &dv, InflateCarry *c, const uint8_t *dict, int32_t len, cudaStream_t cs) {
	if (len < 0 || (len > 0 && !dict)) {
		set_error("buffer/count");
		return B200Z_E_ARG;
	}
	if (!c->need_dict) {
		set_error("Dictionary is not needed"); // InvalidOperationException
		return B200Z_E_STATE;
	}
	uint32_t a = 1;
	if (len > 0) {
		int rc = b200z_adler32(dict, len, &a);
		if (rc) return rc;
	}
	if (a != c->read_adler) {
		set_error("Wrong adler checksum"); // SharpZipBaseException
		return B200Z_E_DATA;
	}
	const int32_t keep = len > (int32_t)kCarryWindow ? (int32_t)kCarryWindow : len; // OutputWindow.CopyDict :160-166
	if (keep > 0) {
		B200Z_CUDA(cudaMemcpyAsync(dv.pool.p + ((int64_t)c->pool + 1) * kCarryWindow - keep, dict + (len - keep), (size_t)keep,
		                           cudaMemcpyHostToDevice, cs));
		B200Z_CUDA(cudaStreamSynchronize(cs));
		dv.h2d += keep;
	}
	c->win_len = keep;
	c->need_dict = false;
	c->adler = 1;
	c->new_input = true; // what was handed over behind the header can be decoded now
	return B200Z_OK;
}

// The Inflater handle: one stream, one plan kept between runs, on the legacy default stream.
struct InflaterH {
	InflateCarry c;
	CarryDevice dv;
	CarryPlan cp;
	int64_t runs = 0; // b200z_inflater_get_stats v[0]
};

// decodes from the resume point to the end of what is available, in runs of the handle's plan until no output capacity
// is outgrown
static int inflater_run_device(InflaterH *d) {
	int rc = d->dv.ensure_pool(1);
	if (rc) return rc;
	const std::vector<InflateCarry *> one{&d->c};
	for (int attempt = 0; attempt < 8; attempt++) {
		if ((rc = inflate_run(d->dv, d->cp, one, 0))) return rc;
		d->runs++;
		if (d->c.out_need == 0) return B200Z_OK;
	}
	set_error("output larger than any capacity tried");
	return B200Z_E_NOMEM;
}

// ---- Inflater set --------------------------------------------------------------------------------------------------
// n Inflater streams of one wrap, driven together: a write appends every stream's piece (SetInput) and runs every stream
// that can go on as plans on the set's CUDA stream.  Due streams are taken in order into plans of at most kInfPlanBytes
// of compressed capacity and kInfPlanOut of output capacity (a stream larger than that runs alone), so one plan's device
// workspace does not grow with the number of streams; the plans are kept and reused while the due streams fit them.
// (The CPU test tier builds the kernels on the CUDA emulator with smaller values, for small data.)
#ifndef B200Z_INFLATE_SET_PLAN_BYTES
#define B200Z_INFLATE_SET_PLAN_BYTES (256ll << 20)
#endif
#ifndef B200Z_INFLATE_SET_PLAN_OUT
#define B200Z_INFLATE_SET_PLAN_OUT (4ll << 30)
#endif
constexpr int64_t kInfPlanBytes = B200Z_INFLATE_SET_PLAN_BYTES;
constexpr int64_t kInfPlanOut = B200Z_INFLATE_SET_PLAN_OUT;

} // namespace b200z

struct b200z_inflate_streams {
	int device = -1, wrap = B200Z_WRAP_ZLIB;
	std::vector<b200z::InflateCarry> s;
	b200z::CarryDevice dv; // window pool of n slots; staging grows to the largest plan
	std::vector<b200z::CarryPlan> plans; // the k-th plan of a round of runs
	cudaStream_t cs = nullptr;
	int broken = 0; // a run failed: the streams' state is not what their output says, no more writes
	int64_t runs = 0, plans_run = 0; // b200z_inflate_streams_stats v[0], v[1]
};

namespace b200z {

// runs every stream that can go on, in rounds: a stream whose output outgrew its capacity goes on in the next round
static int inflate_set_runs(b200z_inflate_streams *S, std::vector<char> &due) {
	const int n = (int)S->s.size();
	for (int round = 0;; round++) {
		std::vector<InflateCarry *> todo;
		for (int i = 0; i < n; i++) {
			InflateCarry *c = &S->s[(size_t)i];
			if (!due[(size_t)i]) continue;
			if (c->attempts >= 8) {
				c->error = B200Z_E_NOMEM; // (output larger than any capacity tried)
				c->attempts = 0;
			}
			if (carry_runs(c) && (round == 0 || c->out_need)) todo.push_back(c);
		}
		if (todo.empty()) return B200Z_OK;
		size_t g = 0;
		for (size_t a = 0; a < todo.size(); g++) {
			std::vector<InflateCarry *> grp;
			int64_t cb = 0, ob = 0;
			for (; a < todo.size(); a++) {
				const int64_t comp = carry_cut(todo[a]).comp, cc = carry_comp_cap(comp);
				const int64_t oc = std::max(carry_out_need(todo[a], comp), cc * 8 + 65536);
				if (!grp.empty() && (cb + cc > kInfPlanBytes || ob + oc > kInfPlanOut)) break;
				cb += cc;
				ob += oc;
				grp.push_back(todo[a]);
			}
			if (S->plans.size() <= g) S->plans.emplace_back();
			int rc = inflate_run(S->dv, S->plans[g], grp, S->cs);
			if (rc) return rc;
			S->runs += (int64_t)grp.size();
			S->plans_run++;
			for (InflateCarry *c : grp) c->note_held();
		}
	}
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
	d->c.wrap = raw ? B200Z_WRAP_RAW : B200Z_WRAP_ZLIB;
	*h = d;
	return B200Z_OK;
}
int b200z_inflater_destroy(void *h) {
	delete (InflaterH *)h;
	return B200Z_OK;
}
int b200z_inflater_reset(void *h) {
	InflaterH *d = (InflaterH *)h;
	d->c.reset();
	d->runs = 0;
	return B200Z_OK;
}
int b200z_inflater_set_dictionary(void *h, const uint8_t *dict, int32_t len) {
	InflaterH *d = (InflaterH *)h;
	int rc = d->c.need_dict ? d->dv.ensure_pool(1) : B200Z_OK;
	return rc ? rc : carry_set_dictionary(d->dv, &d->c, dict, len, 0);
}
int b200z_inflater_set_input(void *h, const uint8_t *buf, int32_t len) {
	InflaterH *d = (InflaterH *)h;
	if (len < 0 || (len > 0 && !buf)) {
		set_error("buffer/count");
		return B200Z_E_ARG;
	}
	if (d->c.in_total > d->c.consumed && !d->c.finished) {
		set_error("Old input was not completely processed"); // StreamManipulator.cs:263
		return B200Z_E_STATE;
	}
	carry_input(&d->c, buf, len);
	return B200Z_OK;
}

static int inflater_error(const InflateCarry &c) {
	set_error("%s", inflate_detail_msg((c.error >> 8) & 0xFF));
	return c.error & 0xFF;
}

int b200z_inflater_inflate(void *h, uint8_t *out, int32_t cap, int32_t *produced) {
	InflaterH *d = (InflaterH *)h;
	InflateCarry &c = d->c;
	if (!produced || cap < 0 || (cap > 0 && !out)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	*produced = 0;
	if (c.error) return inflater_error(c);
	if (!c.finished && c.new_input) {
		c.new_input = false;
		if (!carry_header(&c)) return c.error ? inflater_error(c) : B200Z_OK;
		if (!c.raw_done) {
			int rc = inflater_run_device(d);
			c.note_held();
			if (rc) return rc;
		}
		carry_trailer(&c);
	}
	size_t avail = (size_t)(c.out_total() - c.delivered);
	size_t take = avail < (size_t)cap ? avail : (size_t)cap;
	if (take) memcpy(out, c.output.data() + (c.delivered - c.out_base), take);
	c.delivered += (int64_t)take;
	*produced = (int32_t)take;
	if (take == 0 && c.error) return inflater_error(c);
	return B200Z_OK;
}
int b200z_inflater_needs_input(void *h, int *flag) {
	InflaterH *d = (InflaterH *)h;
	*flag = (d->c.in_total <= d->c.consumed) ? 1 : 0; // StreamManipulator.IsNeedingInput
	return B200Z_OK;
}
int b200z_inflater_needs_dictionary(void *h, int *flag) {
	*flag = ((InflaterH *)h)->c.need_dict ? 1 : 0; // mode == DECODE_DICT && neededBits == 0 (Inflater.cs:792-798)
	return B200Z_OK;
}
int b200z_inflater_is_finished(void *h, int *flag) {
	const InflateCarry &c = ((InflaterH *)h)->c;
	// Inflater.cs:806-812; a trailer that did not verify is an exception from Inflate() in the reference (DecodeChksum
	// :397-418), so the stream is not "finished" as long as that error has not been delivered
	*flag = (c.finished && !c.error && c.delivered == c.out_total()) ? 1 : 0;
	return B200Z_OK;
}
int b200z_inflater_remaining_input(void *h, int32_t *v) {
	const InflateCarry &c = ((InflaterH *)h)->c;
	*v = (int32_t)(c.in_total - c.consumed);
	return B200Z_OK;
}
int b200z_inflater_total_in(void *h, int64_t *v) {
	*v = ((InflaterH *)h)->c.consumed; // totalIn - RemainingInput (Inflater.cs:862-868)
	return B200Z_OK;
}
int b200z_inflater_total_out(void *h, int64_t *v) {
	*v = ((InflaterH *)h)->c.delivered;
	return B200Z_OK;
}
int b200z_inflater_adler(void *h, uint32_t *v) {
	const InflateCarry &c = ((InflaterH *)h)->c;
	*v = c.wrap == B200Z_WRAP_RAW ? 0u : c.adler;
	return B200Z_OK;
}
int b200z_inflater_get_stats(void *h, int64_t *v, int32_t cap) {
	if (!h || cap < 0 || (cap > 0 && !v)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const InflaterH *d = (const InflaterH *)h;
	const int64_t s[4] = {d->runs, d->c.decoded, d->c.max_comp, d->c.max_out};
	for (int32_t i = 0; i < cap && i < 4; i++) v[i] = s[i];
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

int b200z_inflate_streams_create(int32_t n, int wrap, b200z_inflate_streams **s) {
	if (!s || n < 0) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	if (wrap != B200Z_WRAP_RAW && wrap != B200Z_WRAP_ZLIB && wrap != B200Z_WRAP_RAW_CRC32) {
		set_error("wrap: RAW, ZLIB or RAW_CRC32");
		return B200Z_E_ARG;
	}
	int rc = ensure_init();
	if (rc) return rc;
	b200z_inflate_streams *S = new b200z_inflate_streams();
	S->device = current_device();
	DeviceGuard guard(S->device);
	S->wrap = wrap;
	S->s = std::vector<InflateCarry>((size_t)n);
	for (int32_t i = 0; i < n; i++) {
		InflateCarry &c = S->s[(size_t)i];
		c.wrap = wrap;
		c.pool = i;
		c.reset();
	}
	if ((rc = S->dv.ensure_pool(n))) {
		delete S;
		return rc;
	}
	if (cudaStreamCreateWithFlags(&S->cs, cudaStreamNonBlocking) != cudaSuccess) {
		delete S;
		set_error("cudaStreamCreate failed");
		return B200Z_E_CUDA;
	}
	*s = S;
	return B200Z_OK;
}

// a stream's status as a write reports it: its data error, B200Z_E_NEED_INPUT while it is not finished, B200Z_OK after
static int32_t inflate_set_status(const InflateCarry &c) { return c.error ? c.error : (c.finished ? B200Z_OK : B200Z_E_NEED_INPUT); }

int b200z_inflate_streams_write(b200z_inflate_streams *S, const uint8_t *const *in, const int64_t *len, int32_t *status) {
	if (!S || (!S->s.empty() && (!in || !len || !status))) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	const int n = (int)S->s.size();
	for (int i = 0; i < n; i++) // (nothing is taken when an argument is bad)
		if (len[i] < 0 || len[i] > 0x7FFFFFFF || (len[i] > 0 && !in[i])) {
			set_error("stream %d: buffer/count", i);
			return B200Z_E_ARG;
		}
	if (S->broken) {
		set_error("an earlier run of this Inflater set failed with status %d", S->broken);
		return S->broken;
	}
	DeviceGuard guard(S->device);
	std::vector<char> due((size_t)n, 0), late((size_t)n, 0);
	for (int i = 0; i < n; i++) {
		InflateCarry &c = S->s[(size_t)i];
		if (len[i] > 0) {
			if (c.finished) late[(size_t)i] = 1; // "Finish() already called" in the Deflater set: the input is refused
			else if (!c.error) carry_input(&c, in[i], len[i]);
		}
		if (!c.finished && !c.error && c.new_input) {
			c.new_input = false;
			due[(size_t)i] = carry_header(&c) ? 1 : 0;
		}
	}
	const int rc = inflate_set_runs(S, due);
	if (rc) {
		S->broken = rc;
		return rc;
	}
	int first = -1;
	for (int i = 0; i < n; i++) {
		InflateCarry &c = S->s[(size_t)i];
		if (due[(size_t)i]) carry_trailer(&c);
		c.note_held();
		status[i] = late[(size_t)i] ? B200Z_E_STATE : inflate_set_status(c);
		if (first < 0 && status[i] != B200Z_OK && (status[i] & 0xFF) != B200Z_E_NEED_INPUT) first = i;
	}
	if (first < 0) return B200Z_OK;
	if (late[(size_t)first]) set_error("stream %d: input behind the end of the stream", first);
	else set_error("stream %d: %s", first, inflate_detail_msg((status[first] >> 8) & 0xFF));
	return status[first] & 0xFF;
}

int b200z_inflate_streams_read(b200z_inflate_streams *S, uint8_t *const *out, const int64_t *cap, int64_t *got) {
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
		InflateCarry &c = S->s[(size_t)i];
		const int64_t take = std::min<int64_t>(cap[i], c.out_total() - c.delivered);
		if (take > 0) memcpy(out[i], c.output.data() + (c.delivered - c.out_base), (size_t)take);
		c.delivered += take;
		got[i] = take;
	}
	return B200Z_OK;
}

int b200z_inflate_streams_state(b200z_inflate_streams *S, int32_t *flags, int64_t *total_in, int64_t *total_out, int64_t *remaining,
                                int32_t *status) {
	if (!S) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	for (size_t i = 0; i < S->s.size(); i++) {
		const InflateCarry &c = S->s[i];
		if (flags) flags[i] = (c.finished && !c.error ? 1 : 0) | (c.need_dict ? 2 : 0);
		if (total_in) total_in[i] = c.consumed;
		if (total_out) total_out[i] = c.out_total();
		if (remaining) remaining[i] = c.in_total - c.consumed;
		if (status) status[i] = inflate_set_status(c);
	}
	return B200Z_OK;
}

int b200z_inflate_streams_check(b200z_inflate_streams *S, uint32_t *check) {
	if (!S || (!S->s.empty() && !check)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	for (size_t i = 0; i < S->s.size(); i++) {
		const InflateCarry &c = S->s[i];
		check[i] = S->wrap == B200Z_WRAP_RAW ? 0u : (c.need_dict ? c.read_adler : c.run_check);
	}
	return B200Z_OK;
}

int b200z_inflate_streams_set_dictionary(b200z_inflate_streams *S, int32_t i, const uint8_t *dict, int32_t len) {
	if (!S || i < 0 || i >= (int32_t)S->s.size()) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	DeviceGuard guard(S->device);
	return carry_set_dictionary(S->dv, &S->s[(size_t)i], dict, len, S->cs);
}

int b200z_inflate_streams_stats(b200z_inflate_streams *S, int64_t *v, int32_t cap) {
	if (!S || cap < 0 || (cap > 0 && !v)) {
		set_error("bad arguments");
		return B200Z_E_ARG;
	}
	int64_t held = 0;
	for (const InflateCarry &c : S->s) held = std::max(held, c.max_comp);
	const int64_t s[6] = {S->runs, S->plans_run, S->dv.plans_created, held, S->dv.workspace, S->dv.h2d};
	for (int32_t i = 0; i < cap && i < 6; i++) v[i] = s[i];
	return B200Z_OK;
}

int b200z_inflate_streams_destroy(b200z_inflate_streams *S) {
	if (!S) return B200Z_OK;
	DeviceGuard guard(S->device); // (the device buffers and plans go while the set's device is current)
	if (S->cs) {
		cudaStreamSynchronize(S->cs);
		cudaStreamDestroy(S->cs);
	}
	delete S;
	return B200Z_OK;
}

const char *b200z_inflate_detail_message(int32_t status) { return inflate_detail_msg((status >> 8) & 0xFF); }


} // extern "C"
