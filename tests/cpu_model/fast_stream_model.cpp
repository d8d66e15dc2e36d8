// fast_stream_model.cpp -- TEST INFRASTRUCTURE.  model.cpp plus the open runs of levels 0-4 (B200Z_END_NONE): a run entered
// with the engine state of a flush or of the previous run's cut, taking the BUSY_STATE loops of its SetInput calls, writing
// only the blocks the engine closed itself and reporting the engine right behind the last of them.  It runs the serial
// statement in b200z_core.cuh (fe_run / stored_run in their open mode) that k_fast follows warp-cooperatively and that the
// level-0 plan runs when it is built.
#include "model.cpp"

// state: kFastStateBytes (levels 1-4: head[], prev[], FastCarry) or a StoredCarry (level 0), read when cont != 0 and written
// -- behind a flush / finish, or at the cut of an open run (untouched when an open run closes no block).
// cut[2] = covered (data bytes in front of the first block not written, 0 = none closed), SetInput call of the cut.
// end_mode: 0 finish, 1 flush then finish, 2 flush, 3 open.
extern "C" int model_deflate_fast_run(const uint8_t *data, uint32_t n, uint32_t H, uint32_t pos_base, uint32_t bit_base, int level,
                                      int strategy, int end_mode, const uint32_t *cum, int nchunks, int busy_last, uint8_t *state,
                                      int cont, uint8_t *out, uint64_t cap, uint64_t *outbits, int64_t *cut) {
	const LevelParams lp = level_params(level);
	if (lp.func == 2) return 104;
	cut[0] = cut[1] = 0;
	if (end_mode != 3 && lp.func == 1) {
		ModelSched ms;
		ms.cum = cum;
		ms.nchunks = nchunks;
		ms.state = state;
		ms.cont = cont;
		ms.busy_last = busy_last;
		uint64_t len;
		return model_run(data, n, H, pos_base - H, bit_base, nullptr, level, strategy, end_mode == 1, end_mode == 2, out, cap, &len,
		                 outbits, ms);
	}
	Writer W;
	uint64_t bitpos = bit_base;
	if (lp.func == 0) {
		// the level-0 plan when it is built: stored_rebase, then stored_run in any end mode
		StoredCarry cin, cout;
		uint32_t start_bias = 0;
		if (cont) {
			std::memcpy(&cin, state, sizeof cin);
			start_bias = stored_rebase(cin, H);
		}
		int call = 0;
		uint32_t end = H;
		stored_run(n - H, cont ? 0 : H, end_mode, [&](uint32_t start, uint32_t len, bool last) {
			W.put(bitpos, last ? 1 : 0, 3);
			bitpos = (bitpos + 3 + 7) & ~7ull;
			W.put(bitpos, len & 0xFFFF, 16);
			W.put(bitpos + 16, (~len) & 0xFFFF, 16);
			bitpos += 32;
			for (uint32_t i = 0; i < len; i++, bitpos += 8) W.put(bitpos, data[start + i], 8);
			end = start + len;
		}, cum, nchunks, cont ? &cin : nullptr, &cout, start_bias, busy_last != 0, &call);
		std::memcpy(state, &cout, sizeof cout);
		if (end_mode == 3) {
			cut[0] = end - H;
			cut[1] = call;
		}
	} else {
		std::vector<uint16_t> head(32768, 0), prev(32768, 0);
		FastEngine fe;
		if (cont) {
			FastCarry c;
			std::memcpy(head.data(), state, 65536);
			std::memcpy(prev.data(), state + 65536, 65536);
			std::memcpy(&c, state + 131072, sizeof c);
			fe_load(fe, c, data, n, H, head.data(), prev.data());
		} else {
			fe_init(fe, data, n, head.data(), prev.data());
			fe_set_dictionary(fe, H);
		}
		std::vector<uint32_t> syms, blk_start;
		std::vector<bool> blk_ok;
		size_t nblocks = 0;
		fe_run(fe, lp, strategy, 3, [&](uint32_t sym) { syms.push_back(sym); },
		       [&](uint32_t start, bool ok, bool) {
			       blk_start.push_back(start);
			       blk_ok.push_back(ok);
		       },
		       [&](int ci) {
			       // the engine right behind the block that just closed
			       FastCarry c;
			       fe_save(fe, c);
			       std::memcpy(state, head.data(), 65536);
			       std::memcpy(state + 65536, prev.data(), 65536);
			       std::memcpy(state + 131072, &c, sizeof c);
			       nblocks = blk_start.size();
			       cut[0] = (int64_t)((uint32_t)fe.blockStart + fe.woff) - H;
			       cut[1] = ci;
		       },
		       cum, nchunks, true);
		blk_start.resize(nblocks);
		blk_start.push_back((uint32_t)(cut[0] + H));
		std::vector<int> scratch(kTreeScratchInts + 64);
		for (size_t b = 0; b < nblocks; b++) {
			int lit_freqs[kLiteralNum] = {0}, dist_freqs[kDistNum] = {0};
			int extra = 0;
			for (size_t i = b * kBlockSyms; i < (b + 1) * kBlockSyms; i++) {
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
			uint8_t lit_len[kLiteralNum], dist_len[kDistNum];
			uint16_t lit_codes[kLiteralNum], dist_codes[kDistNum];
			uint32_t hdr[192];
			std::memset(hdr, 0, sizeof(hdr));
			BlockPlan plan;
			plan_block(lit_freqs, dist_freqs, extra, blk_ok[b], (int)blen, 0, lit_len, lit_codes, dist_len, dist_codes, hdr,
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
				for (size_t i = b * kBlockSyms; i < (b + 1) * kBlockSyms; i++) {
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
	}
	*outbits = bitpos;
	const uint64_t nbytes = (bitpos + 7) >> 3;
	if (nbytes > cap) return 102;
	W.w.resize((nbytes + 3) / 4 + 1, 0);
	std::memcpy(out, W.w.data(), nbytes);
	return 0;
}
