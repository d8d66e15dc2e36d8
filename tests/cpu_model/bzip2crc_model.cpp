// TEST INFRASTRUCTURE: BZip2Crc (Checksum/BZip2Crc.cs:43-170) restated over CrcUtilities (CrcUtilities.cs:25-77, 134-156),
// the reference the CRC-32/BZIP2 kernel (kind 2 of b200z_checksum.cu) is held against.  It walks the bytes the way the
// reference does: 16 slicing tables made for the normal polynomial, 16-byte steps through UpdateDataForNormalPoly, and the
// bytes that do not fill a step through Update(int).  Never linked into the product.
#include <cstddef>
#include <cstdint>

namespace {

constexpr int kSlicingDegree = 16;           // CrcUtilities.SlicingDegree
constexpr uint32_t kPoly = 0x04C11DB7u;      // BZip2Crc.crcTable's polynomial
constexpr uint32_t kCrcInit = 0xFFFFFFFFu;   // BZip2Crc.crcInit

struct Table {
	uint32_t t[256 * kSlicingDegree];
	// GenerateSlicingLookupTable(polynomial, isReversed: false): the byte starts in the top 8 bits and every slice takes it
	// 8 more steps; a step shifts left and folds the polynomial in when the bit shifted out (bit 31) was set
	Table() {
		for (uint32_t i = 0; i < 256; i++) {
			uint32_t res = i << 24;
			for (int j = 0; j < kSlicingDegree; j++) {
				for (int k = 0; k < 8; k++) res = (res & 0x80000000u) != 0 ? kPoly ^ (res << 1) : res << 1;
				t[256 * j + i] = res;
			}
		}
	}
};

const Table &table() {
	static const Table tab;
	return tab;
}

// UpdateDataForNormalPoly: the register's bytes, top first, mix into the first four input bytes; then UpdateDataCommon
// looks up input byte k of the 16 in slice 15 - k
uint32_t update_data_for_normal_poly(const uint8_t *in, uint32_t check) {
	const uint32_t *t = table().t;
	const uint8_t x1 = (uint8_t)((uint8_t)(check >> 24) ^ in[0]);
	const uint8_t x2 = (uint8_t)((uint8_t)(check >> 16) ^ in[1]);
	const uint8_t x3 = (uint8_t)((uint8_t)(check >> 8) ^ in[2]);
	const uint8_t x4 = (uint8_t)((uint8_t)check ^ in[3]);
	uint32_t r = t[x1 + 256 * 15] ^ t[x2 + 256 * 14] ^ t[x3 + 256 * 13] ^ t[x4 + 256 * 12];
	for (int k = 4; k < 16; k++) r ^= t[in[k] + 256 * (15 - k)];
	return r;
}

// BZip2Crc.Update(int bval): the low 8 bits of bval against the register's top byte
uint32_t update_int(uint32_t check, int bval) {
	return table().t[(uint8_t)(((check >> 24) & 0xFF) ^ (uint32_t)bval)] ^ (check << 8);
}

// BZip2Crc.Update(byte[] data, int offset, int count): whole 16-byte steps, then SlowUpdateLoop over the rest
uint32_t update_span(uint32_t check, const uint8_t *data, int32_t count) {
	const int32_t remainder = count % kSlicingDegree;
	const int32_t end = count - remainder;
	int32_t offset = 0;
	while (offset != end) {
		check = update_data_for_normal_poly(data + offset, check);
		offset += kSlicingDegree;
	}
	while (offset != end + remainder) check = update_int(check, data[offset++]);
	return check;
}

} // namespace

extern "C" {

// Value after Update(data[0 .. n)) on a BZip2Crc whose Value was `value` (checkValue = ~value; Reset -> value 0).  An array
// holds at most 2^31 - 1 bytes in the reference, so a longer span is fed as several Updates of at most 1 GiB each.
uint32_t bz2crc_model_update(uint32_t value, const uint8_t *data, uint64_t n) {
	uint32_t check = ~value;
	for (uint64_t p = 0; p < n;) {
		const uint64_t piece = n - p < (1ull << 30) ? n - p : (1ull << 30);
		check = update_span(check, data + p, (int32_t)piece);
		p += piece;
	}
	return ~check;
}

// Value after Update(int bval) on a BZip2Crc whose Value was `value`
uint32_t bz2crc_model_update_int(uint32_t value, int32_t bval) { return ~update_int(~value, bval); }

// Value of a new BZip2Crc: Reset() sets checkValue to crcInit, and Value is ~checkValue
uint32_t bz2crc_model_reset_value(void) { return ~kCrcInit; }

} // extern "C"
