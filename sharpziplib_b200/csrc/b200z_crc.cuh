// b200z_crc.cuh -- GF(2) arithmetic for the tile-parallel CRC-32 and CRC-32/BZIP2, and the modular arithmetic for Adler-32.
//
// The reference walks the buffer serially (Crc32.Update, Checksum/Crc32.cs:138-159, and BZip2Crc.Update,
// Checksum/BZip2Crc.cs:136-169, slicing-by-16 in CrcUtilities.cs:69-156; Adler32.Update, Checksum/Adler32.cs:134-161).  All
// three checksums are linear, so the device computes one partial per 128-byte chunk and combines partials with the identities
// below.  Same result, bit for bit.
//
// CRC-32 (reflected 0xEDB88320) and CRC-32/BZIP2 (normal 0x04C11DB7).  raw(s, D) = register after feeding D starting from
// register s, no final xor.  In either bit order:
//   raw(s, D) = shift(s, |D|) ^ raw(0, D),   shift(s, L) = s * x^(8L) mod P          (feeding L zero bytes)
//   raw(0, A || B) = shift(raw(0, A), |B|) ^ raw(0, B)
//   Value after Update(M) from value v0:  (shift(v0 ^ ~0, |M|) ^ raw(0, M)) ^ ~0     (init = xorout = ~0 for both)
// The bit orders differ in where x^0 sits and how a byte enters.  Reflected (crc_*): x^0 is bit 31, the register shifts
// right, and a byte enters at the bottom, least significant bit first.  Normal (crcn_*): x^0 is bit 0, the register shifts
// left, and a byte enters at the top, most significant bit first, so a little-endian word is byte-swapped before it is fed.
// Adler-32 (mod 65521), from (s1, s2):  s1' = s1 + sum b_i,  s2' = s2 + n*s1 + sum (n - i) * b_i.
#pragma once
#include "b200z_core.cuh"

namespace b200z {

constexpr uint32_t kCrcPoly = 0xEDB88320u;
constexpr uint32_t kCrcnPoly = 0x04C11DB7u; // CRC-32/BZIP2 (BZip2Crc.cs:50)
constexpr uint32_t kAdlerBase = 65521u;
constexpr int kCkChunk = 128;                 // bytes per thread
constexpr int kCkThreads = 256;               // threads per tile
constexpr int kCkTile = kCkChunk * kCkThreads; // 32 KiB

// a(x) * b(x) mod P in the reflected representation (x^0 = 0x80000000)
B200Z_HD uint32_t crc_mulmod(uint32_t a, uint32_t b) {
	uint32_t p = 0;
#ifdef __CUDA_ARCH__
#pragma unroll 8
#endif
	for (int i = 0; i < 32; i++) { // fixed trip count: cannot spin on a == 0
		if (a & (0x80000000u >> i)) p ^= b;
		b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
	}
	return p;
}

// x^(8 * nbytes) mod P by square-and-multiply
B200Z_HDN uint32_t crc_xpow8(uint64_t nbytes) {
	uint32_t p = 1u << 31;         // x^0
	uint32_t sq = 1u << 23;        // x^8: bit (31 - 8)
	// x^8 in reflected form is 0x00800000
	while (nbytes) {
		if (nbytes & 1) p = crc_mulmod(sq, p);
		sq = crc_mulmod(sq, sq);
		nbytes >>= 1;
	}
	return p;
}

// byte-at-a-time table entry (CrcUtilities.GenerateSlicingLookupTable :25-52, slice 0)
B200Z_HD uint32_t crc_table0_entry(uint32_t i) {
	uint32_t res = i;
	for (int k = 0; k < 8; k++) res = (res & 1) ? kCrcPoly ^ (res >> 1) : res >> 1;
	return res;
}

// a(x) * b(x) mod P in the normal representation (x^0 = 0x00000001)
B200Z_HD uint32_t crcn_mulmod(uint32_t a, uint32_t b) {
	uint32_t p = 0;
#ifdef __CUDA_ARCH__
#pragma unroll 8
#endif
	for (int i = 0; i < 32; i++) { // fixed trip count: cannot spin on a == 0
		if (a & (1u << i)) p ^= b;
		b = (b & 0x80000000u) ? (b << 1) ^ kCrcnPoly : b << 1;
	}
	return p;
}

// x^(8 * nbytes) mod P, normal representation, by square-and-multiply
B200Z_HDN uint32_t crcn_xpow8(uint64_t nbytes) {
	uint32_t p = 1u;       // x^0
	uint32_t sq = 1u << 8; // x^8
	while (nbytes) {
		if (nbytes & 1) p = crcn_mulmod(sq, p);
		sq = crcn_mulmod(sq, sq);
		nbytes >>= 1;
	}
	return p;
}

// byte-at-a-time table entry for the normal polynomial (GenerateSlicingLookupTable with isReversed: false, slice 0)
B200Z_HD uint32_t crcn_table0_entry(uint32_t i) {
	uint32_t res = i << 24;
	for (int k = 0; k < 8; k++) res = (res & 0x80000000u) ? kCrcnPoly ^ (res << 1) : res << 1;
	return res;
}

struct CkTile {
	uint64_t start; // first byte of the tile inside its stream (64-bit: a stream may be longer than 4 GiB)
	int32_t stream;
	uint32_t mult;  // CRCs: x^(8 * bytes after this tile) in the kind's bit order ; Adler: bytes after this tile mod 65521
};
static_assert(sizeof(CkTile) == 16, "one tile descriptor per 16 bytes");

} // namespace b200z
