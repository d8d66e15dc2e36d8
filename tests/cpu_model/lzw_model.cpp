// lzw_model.cpp -- TEST INFRASTRUCTURE for the LZW (.Z) decoder: a restatement of SharpZipLib's LzwInputStream
// (Lzw/LzwInputStream.cs) with its 8 KiB buffer, Fill() and group-wise bitIn, over a base stream whose Read() returns as
// many bytes as the caller's schedule says; and a compress(1)-format encoder written from the format.  Never linked into
// the product.  Built by tests/lzw_ref.py.
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace {

// What the reference throws, as (kind, a, b):
//   1 "Wrong LZW header. Magic bytes don't match. 0x<a> 0x<b>"
//   2 "Stream compressed with <a> bits, but decompression can only handle 16 bits."
//   3 "Unsupported bits set in the header."
//   4 "corrupt input: <a> > 255"
//   5 "corrupt input: code=<a>, freeEnt=<b>"
//   6 a non-SharpZip exception (an index outside an array, Array.Copy with a negative length); a says where:
//     1 the header's table initialisation, 2 ResetBuf, 3 the code read, 4 the string tables, 5 the stack
struct Throw {
	int kind, a, b;
};

struct BaseStream {
	const uint8_t *p;
	int64_t len, pos = 0;
	const int32_t *sizes;
	int n_sizes, next = 0;
	int Read(uint8_t *buf, int off, int count) {
		int64_t k = count;
		if (n_sizes > 0) {
			const int64_t s = sizes[next];
			next = (next + 1) % n_sizes;
			if (s < k) k = s;
		}
		if (k > len - pos) k = len - pos;
		if (k < 0) k = 0;
		memcpy(buf + off, p + pos, (size_t)k);
		pos += k;
		return (int)k;
	}
};

struct Lzw {
	BaseStream *base;
	bool headerParsed = false, eof = false, blockMode = false;
	std::vector<int> tabPrefix;
	std::vector<uint8_t> tabSuffix, stack;
	int nBits = 0, maxBits = 0, maxMaxCode = 0, maxCode = 0, bitMask = 0, oldCode = 0, stackP = 0, freeEnt = 0;
	uint8_t finChar = 0;
	uint8_t data[8192] = {};
	int bitPos = 0, end = 0, got = 0;
	static constexpr int EXTRA = 64;
	int thrown_after = 0; // bytes the Read that threw had written into the caller's buffer

	int ResetBuf(int bitPosition) {
		const int pos = bitPosition >> 3;
		if (end - pos < 0 || pos > (int)sizeof(data)) throw Throw{6, 2, 0};
		memmove(data, data + pos, (size_t)(end - pos));
		end -= pos;
		return 0;
	}
	void Fill() {
		got = base->Read(data, end, (int)sizeof(data) - 1 - end);
		if (got > 0) end += got;
	}
	void ParseHeader() {
		headerParsed = true;
		uint8_t hdr[3] = {0, 0, 0};
		base->Read(hdr, 0, 3); // one Read: a short read leaves zeros
		if (hdr[0] != 0x1F || hdr[1] != 0x9D) throw Throw{1, hdr[0], hdr[1]};
		blockMode = (hdr[2] & 0x80) > 0;
		maxBits = hdr[2] & 0x1F;
		if (maxBits > 16) throw Throw{2, maxBits, 0};
		if (hdr[2] & 0x60) throw Throw{3, 0, 0};
		maxMaxCode = 1 << maxBits;
		nBits = 9;
		maxCode = (1 << nBits) - 1;
		bitMask = maxCode;
		oldCode = -1;
		finChar = 0;
		freeEnt = blockMode ? 257 : 256;
		tabPrefix.assign((size_t)1 << maxBits, 0);
		tabSuffix.assign((size_t)1 << maxBits, 0);
		stack.assign((size_t)1 << maxBits, 0);
		stackP = (int)stack.size();
		if (tabSuffix.size() < 256) throw Throw{6, 1, 0}; // tabSuffix[255] = 255
		for (int idx = 255; idx >= 0; idx--) tabSuffix[(size_t)idx] = (uint8_t)idx;
	}
	uint8_t suffix(int c) {
		if (c < 0 || c >= (int)tabSuffix.size()) throw Throw{6, 4, 0};
		return tabSuffix[(size_t)c];
	}
	int prefix(int c) {
		if (c < 0 || c >= (int)tabPrefix.size()) throw Throw{6, 4, 0};
		return tabPrefix[(size_t)c];
	}
	void push(uint8_t v) {
		if (stackP <= 0) throw Throw{6, 5, 0};
		stack[(size_t)--stackP] = v;
	}

	// Read(buffer, offset, count) of the reference; the locals are written back only where it writes them back
	int Read(uint8_t *buffer, int offset, int count) {
		if (!headerParsed) ParseHeader();
		if (eof) return 0;
		const int start = offset;
		int lNBits = nBits, lMaxCode = maxCode, lMaxMaxCode = maxMaxCode, lBitMask = bitMask, lOldCode = oldCode;
		uint8_t lFinChar = finChar;
		int lStackP = stackP, lFreeEnt = freeEnt, lBitPos = bitPos;
		const int SL = (int)stack.size();
		int sSize = SL - lStackP;
		if (sSize > 0) {
			const int num = sSize >= count ? count : sSize;
			memcpy(buffer + offset, stack.data() + lStackP, (size_t)num);
			offset += num;
			count -= num;
			lStackP += num;
		}
		if (count == 0) {
			stackP = lStackP;
			return offset - start;
		}
		auto save = [&] {
			nBits = lNBits, maxCode = lMaxCode, maxMaxCode = lMaxMaxCode, bitMask = lBitMask, oldCode = lOldCode;
			finChar = lFinChar, stackP = lStackP, freeEnt = lFreeEnt, bitPos = lBitPos;
		};
		try {
		do {
		main_loop:
			if (end < EXTRA) Fill();
			const int bitIn = got > 0 ? (end - end % lNBits) << 3 : (end << 3) - (lNBits - 1);
			while (lBitPos < bitIn) {
				if (count == 0) {
					save();
					return offset - start;
				}
				if (lFreeEnt > lMaxCode) {
					const int nBytes = lNBits << 3;
					lBitPos = (lBitPos - 1) + nBytes - (lBitPos - 1 + nBytes) % nBytes;
					lNBits++;
					lMaxCode = lNBits == maxBits ? lMaxMaxCode : (1 << lNBits) - 1;
					lBitMask = (1 << lNBits) - 1;
					lBitPos = ResetBuf(lBitPos);
					goto main_loop;
				}
				const int pos = lBitPos >> 3;
				if (pos + 2 >= (int)sizeof(data)) throw Throw{6, 3, 0};
				int code = ((data[pos] | (data[pos + 1] << 8) | (data[pos + 2] << 16)) >> (lBitPos & 7)) & lBitMask;
				lBitPos += lNBits;
				if (lOldCode == -1) {
					if (code >= 256) throw Throw{4, code, 0};
					lFinChar = (uint8_t)(lOldCode = code);
					buffer[offset++] = lFinChar;
					count--;
					continue;
				}
				if (code == 256 && blockMode) {
					std::fill(tabPrefix.begin(), tabPrefix.begin() + 256, 0);
					lFreeEnt = 256;
					const int nBytes = lNBits << 3;
					lBitPos = (lBitPos - 1) + nBytes - (lBitPos - 1 + nBytes) % nBytes;
					lNBits = 9;
					lMaxCode = (1 << lNBits) - 1;
					lBitMask = lMaxCode;
					lBitPos = ResetBuf(lBitPos);
					goto main_loop;
				}
				const int inCode = code;
				lStackP = SL;
				stackP = lStackP;
				if (code >= lFreeEnt) {
					if (code > lFreeEnt) throw Throw{5, code, lFreeEnt};
					stackP = lStackP;
					push(lFinChar);
					lStackP = stackP;
					code = lOldCode;
				}
				stackP = lStackP;
				while (code >= 256) {
					push(suffix(code));
					code = prefix(code);
				}
				lStackP = stackP;
				lFinChar = suffix(code);
				buffer[offset++] = lFinChar;
				count--;
				sSize = SL - lStackP;
				const int num = sSize >= count ? count : sSize;
				memcpy(buffer + offset, stack.data() + lStackP, (size_t)num);
				offset += num;
				count -= num;
				lStackP += num;
				if (lFreeEnt < lMaxMaxCode) {
					tabPrefix[(size_t)lFreeEnt] = lOldCode;
					tabSuffix[(size_t)lFreeEnt] = lFinChar;
					lFreeEnt++;
				}
				lOldCode = inCode;
				if (count == 0) {
					save();
					return offset - start;
				}
			}
			lBitPos = ResetBuf(lBitPos);
		} while (got > 0);
		} catch (const Throw &) {
			thrown_after = offset - start;
			throw;
		}
		save();
		eof = true;
		return offset - start;
	}
};

} // namespace

extern "C" {

// Decodes `in` as LzwInputStream does when the caller reads out_chunk bytes per Read (0: everything that fits) and the
// base stream returns at most sizes[k % n_sizes] bytes on its k-th Read after the header (n_sizes 0: no limit).  Writes
// up to cap bytes to out.  delivered = bytes the successful Reads returned, decoded = those plus what the throwing Read
// had decoded when it threw (the bytes in front of the failing code).  Returns the Throw kind (0: no exception).
int lzw_model_decode(const uint8_t *in, int64_t len, const int32_t *sizes, int32_t n_sizes, int64_t out_chunk, uint8_t *out,
                     int64_t cap, int64_t *delivered, int64_t *decoded, int32_t *a, int32_t *b) {
	BaseStream bs{in, len, 0, sizes, n_sizes};
	Lzw z;
	z.base = &bs;
	std::vector<uint8_t> buf;
	int64_t total = 0;
	*a = *b = 0;
	const int chunk = out_chunk > 0 && out_chunk < (1 << 30) ? (int)out_chunk : (1 << 20);
	buf.resize((size_t)chunk);
	for (;;) {
		int r;
		try {
			// the header's Read comes first and takes no schedule entry
			if (!z.headerParsed) {
				bs.n_sizes = 0;
				z.ParseHeader();
				bs.n_sizes = n_sizes;
			}
			r = z.Read(buf.data(), 0, chunk);
		} catch (const Throw &t) {
			*delivered = total;
			*decoded = total + z.thrown_after;
			*a = t.a;
			*b = t.b;
			return t.kind;
		}
		if (r <= 0) break;
		if (total + r <= cap) memcpy(out + total, buf.data(), (size_t)r);
		total += r;
	}
	*delivered = *decoded = total;
	return 0;
}

// compress(1) format.  block: block mode (CLEAR allowed); clear_every > 0: a CLEAR behind every clear_every data codes;
// ratio_clear: the compress(1) checkpoint (every 10000 input bytes once the table is full, CLEAR when the ratio fell).
// Returns the stream length, or the length it needs when cap is too small.
int64_t lzw_model_encode(const uint8_t *in, int64_t len, int max_bits, int block, int64_t clear_every, int ratio_clear, uint8_t *out,
                         int64_t cap) {
	const int maxmax = 1 << max_bits;
	std::vector<int> codes;
	std::unordered_map<uint32_t, int> dict;
	int enc_free = block ? 257 : 256;
	int64_t since_clear = 0, checkpoint = 10000, bits_est = 0;
	int64_t ratio = 0;
	int w = -1;
	auto emit = [&](int c) {
		codes.push_back(c);
		bits_est += 16;
	};
	for (int64_t i = 0; i < len; i++) {
		const int c = in[i];
		if (w < 0) {
			w = c;
			continue;
		}
		const uint32_t key = ((uint32_t)w << 8) | (uint32_t)c;
		auto it = dict.find(key);
		if (it != dict.end()) {
			w = it->second;
			continue;
		}
		emit(w);
		++since_clear;
		bool clear = false;
		if (enc_free < maxmax) {
			dict[key] = enc_free++;
		} else if (block && ratio_clear && i >= checkpoint) {
			checkpoint = i + 10000;
			const int64_t r = bits_est ? (i << 8) / (bits_est / 8 + 1) : 0;
			if (r > ratio) ratio = r;
			else clear = true, ratio = 0;
		}
		if (block && clear_every > 0 && since_clear >= clear_every) clear = true;
		if (clear) {
			emit(256);
			dict.clear();
			enc_free = 257;
			since_clear = 0;
		}
		w = c;
	}
	if (w >= 0) emit(w);
	// pack with the decoder's rules: the width grows before a code when its freeEnt passed maxCode, padded to a whole group
	std::vector<uint8_t> o = {0x1F, 0x9D, (uint8_t)(max_bits | (block ? 0x80 : 0))};
	int64_t bit = 0, group_start = 0; // bits from the first code byte; where the current width began
	int n = 9, maxcode = 511, free_ent = block ? 257 : 256;
	bool first = true;
	auto pad = [&] {
		const int64_t g = (int64_t)n * 8;
		const int64_t rel = bit - group_start;
		bit = group_start + (rel + g - 1) / g * g;
		group_start = bit;
	};
	auto put = [&](int c) {
		const size_t need = (size_t)((bit + n + 7) / 8) + 3;
		if (o.size() < need) o.resize(need, 0);
		for (int k = 0; k < n; k++)
			if ((c >> k) & 1) o[3 + (size_t)((bit + k) >> 3)] |= (uint8_t)(1u << ((bit + k) & 7));
		bit += n;
	};
	for (int c : codes) {
		if (free_ent > maxcode) {
			pad();
			n++;
			maxcode = n == max_bits ? maxmax : (1 << n) - 1;
		}
		put(c);
		if (first) {
			first = false;
			continue;
		}
		if (c == 256 && block) {
			pad();
			n = 9;
			maxcode = 511;
			free_ent = 256;
			continue;
		}
		if (free_ent < maxmax) free_ent++;
	}
	o.resize(3 + (size_t)((bit + 7) / 8));
	if ((int64_t)o.size() <= cap) memcpy(out, o.data(), o.size());
	return (int64_t)o.size();
}

} // extern "C"
