// stream_model.cpp -- TEST INFRASTRUCTURE.  model.cpp plus the open runs of levels 5-9 (B200Z_END_NONE): a run entered with
// a carried parse state, stopped at the last loop top with MIN_LOOKAHEAD bytes ahead, writing only the blocks the
// 16384-symbol rule closed, and reporting where its last block ended and the state there.  The parse here is one serial
// pass (parse_run over the whole run, the state read at every cut), not the kernels' rounds and their re-parse of the
// round that holds the cut, so the two decompositions check each other.
#include "model.cpp"

// entry[3] = prev_available, match_len, match_dist (b200z_parse_entry); cut[4] = covered, and the entry of the next run.
// end_mode: 0 finish, 1 flush then finish, 2 flush, 3 open.  Levels 5-9 only.
extern "C" int model_deflate_open(const uint8_t *data, uint32_t n, uint32_t H, uint32_t pos_base, uint32_t bit_base,
                                  const uint8_t *hmask, int level, int strategy, int end_mode, const int64_t *entry, uint8_t *out,
                                  uint64_t cap, uint64_t *outbits, int64_t *cut) {
	const LevelParams lp = level_params(level);
	if (lp.func != 2) return 104;
	const uint32_t abs_bias = pos_base - H;
	std::vector<uint16_t> link;
	model_links(data, n, link, H, hmask);
	std::vector<uint32_t> tabA(n, 0), tabB(n, 0);
	if (strategy != 2)
		for (uint32_t p = H; p < n; p++) match_search(data, link.data(), 0u, p, n, lp, tabA[p], tabB[p], abs_bias);
	auto tabf = [&](uint32_t p, uint32_t &a, uint32_t &b) { a = tabA[p]; b = tabB[p]; };
	auto bytef = [&](uint32_t q) { return (uint32_t)data[q]; };
	auto slowf = [&](uint32_t p, uint32_t m0, uint32_t budget) { return match_search_above(data, link.data(), p, n, m0, budget, abs_bias); };
	ParseCarry c;
	c.st.prevAvail = (uint32_t)entry[0];
	c.st.p = H + c.st.prevAvail;
	c.st.mlen = (uint32_t)entry[1];
	c.st.mstart = entry[1] >= kMinMatch ? (uint32_t)(H - entry[2]) : 0u;
	c.last_top = H;
	ParseCarry at_cut = c;
	const uint32_t pend = end_mode == 3 ? (n >= 262 ? n - 261 : 0u) : n;
	std::vector<uint32_t> syms, blk_start(1, H), blk_ptop;
	parse_run<true>(c, pend, n, lp, strategy, tabf, bytef, slowf, [&](uint32_t k, uint32_t sym, uint32_t top, uint32_t bytes_after) {
		syms.push_back(sym);
		if (((k + 1) & (kBlockSyms - 1)) == 0) {
			blk_ptop.push_back(top);
			blk_start.push_back(bytes_after);
			at_cut = c; // parse_run calls emit right behind the step that tallied the symbol
		}
	});
	size_t nblocks = blk_ptop.size();
	if (end_mode == 3) {
		syms.resize(nblocks * kBlockSyms);
	} else if (!(end_mode == 0 && !syms.empty() && syms.size() % kBlockSyms == 0 && !c.st.prevAvail)) {
		if (c.st.prevAvail) syms.push_back(sym_lit(data[c.st.p - 1])); // final flush at lookahead == 0 (:750-768)
		blk_ptop.push_back(c.last_top);
		blk_start.push_back(n);
		++nblocks;
	}
	const int64_t pos = (int64_t)at_cut.st.p - at_cut.st.prevAvail;
	cut[0] = pos - H;
	cut[1] = at_cut.st.prevAvail;
	cut[2] = at_cut.st.mlen;
	cut[3] = at_cut.st.mlen >= (uint32_t)kMinMatch ? pos - (int64_t)at_cut.st.mstart : 0;
	Writer W;
	uint64_t bitpos = bit_base;
	std::vector<int> scratch(kTreeScratchInts + 64);
	for (size_t b = 0; b < nblocks; b++) {
		const size_t s0 = b * (size_t)kBlockSyms, s1 = s0 + kBlockSyms < syms.size() ? s0 + kBlockSyms : syms.size();
		int lit_freqs[kLiteralNum] = {0}, dist_freqs[kDistNum] = {0};
		int extra = 0;
		for (size_t i = s0; i < s1; i++) {
			const uint32_t s = syms[i];
			if (sym_dist(s) == 0) lit_freqs[s & 0xFF]++;
			else {
				const int lc = lcode((int)(s & 0xFF)), dc = dcode((int)sym_dist(s) - 1);
				lit_freqs[lc]++;
				dist_freqs[dc]++;
				extra += tally_extra_bits(lc, dc);
			}
		}
		lit_freqs[256]++;
		const uint32_t blen = blk_start[b + 1] - blk_start[b];
		const bool last = b + 1 == nblocks && end_mode == 0;
		const int64_t storedOffset = (int64_t)blk_start[b] + abs_bias + 1 - 32768ll * (int64_t)slides_done(blk_ptop[b] + abs_bias);
		uint8_t lit_len[kLiteralNum], dist_len[kDistNum];
		uint16_t lit_codes[kLiteralNum], dist_codes[kDistNum];
		uint32_t hdr[192];
		std::memset(hdr, 0, sizeof(hdr));
		BlockPlan plan;
		plan_block(lit_freqs, dist_freqs, extra, storedOffset >= 0, (int)blen, last, lit_len, lit_codes, dist_len, dist_codes, hdr,
		           scratch.data(), plan);
		if (plan.type == 0) {
			W.put(bitpos, hdr[0], 3);
			bitpos = (bitpos + 3 + 7) & ~7ull;
			W.put(bitpos, blen & 0xFFFF, 16);
			W.put(bitpos + 16, (~blen) & 0xFFFF, 16);
			bitpos += 32;
			for (uint32_t i = 0; i < blen; i++, bitpos += 8) W.put(bitpos, data[blk_start[b] + i], 8);
		} else {
			for (uint32_t i = 0; i < plan.hdr_bits; i += 32) {
				const int nb = plan.hdr_bits - i < 32 ? (int)(plan.hdr_bits - i) : 32;
				W.put(bitpos + i, hdr[i >> 5] & (nb == 32 ? 0xFFFFFFFFu : ((1u << nb) - 1)), nb);
			}
			bitpos += plan.hdr_bits;
			for (size_t i = s0; i < s1; i++) {
				uint64_t bits;
				int nb;
				encode_symbol(syms[i], lit_codes, lit_len, dist_codes, dist_len, bits, nb);
				W.put(bitpos, bits, nb);
				bitpos += nb;
			}
			W.put(bitpos, lit_codes[256], lit_len[256]);
			bitpos += lit_len[256];
		}
	}
	if (end_mode == 1 || end_mode == 2) { // sync padding (Deflater.cs:486-504), then Finish's empty static block
		for (int need = 8 + (int)((0 - bitpos) & 7); need > 0; need -= 10, bitpos += 10) W.put(bitpos, 2, 10);
		if (end_mode == 1) {
			W.put(bitpos, 3, 10);
			bitpos += 10;
		}
	}
	*outbits = bitpos;
	const uint64_t nbytes = (bitpos + 7) >> 3;
	if (nbytes > cap) return 102;
	W.w.resize((nbytes + 3) / 4 + 1, 0);
	std::memcpy(out, W.w.data(), nbytes);
	return 0;
}
