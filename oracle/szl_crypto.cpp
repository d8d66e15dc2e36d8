// szl_crypto.cpp -- ORACLE (test infrastructure; never linked into the product): CPU restatement of the reference's
// two entry ciphers, SURVEY.md row f4.  Paths are relative to SharpZipLib's src/ICSharpCode.SharpZipLib/.
//
//   Encryption/ZipAESTransform.cs  :41-72  constructor: PBKDF2-HMAC-SHA1 (1000 rounds) -> key1 | key2 | 2-byte verifier
//                                  :75-112 TransformBlock: AES-CTR, little-endian counter starting at 1, HMAC-SHA1 of the
//                                          ciphertext (of the input when reading, of the output when writing)
//                                  :117-122 PwdVerifier, GetAuthCode (the streams keep the first 10 bytes)
//   Encryption/PkzipClassic.cs     :19-50  GenerateKeys, :74-111 TransformByte / UpdateKeys, :170-178 / :279-288 TransformBlock
//
// The reference takes AES / SHA-1 / HMAC / PBKDF2 from System.Security.Cryptography; they are restated here from their
// public specifications (FIPS 197, FIPS 180-4, RFC 2104, RFC 2898) in the plainest form (S-box AES, one byte at a time) --
// a different formulation from the product's T-table kernels.  Pinned by tests/test_oracle.py against the FIPS-197 /
// RFC 3174 / RFC 6070 known answers, against Python's `cryptography` and `zipfile`, and against the AES-encrypted archive the
// reference's own tests hold (test/.../Zip/ZipEncryptionHandling.cs:452-456).
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

// ---- AES (FIPS 197), encryption direction only (CTR) ------------------------------------------------
uint8_t g_sbox[256];
bool g_sbox_ready = false;
uint8_t gmul(uint8_t a, uint8_t b) {
	uint8_t p = 0;
	for (int i = 0; i < 8; i++) {
		if (b & 1) p ^= a;
		const bool hi = a & 0x80;
		a <<= 1;
		if (hi) a ^= 0x1B;
		b >>= 1;
	}
	return p;
}
void make_sbox() {
	if (g_sbox_ready) return;
	// multiplicative inverse followed by the affine map (FIPS 197 5.1.1)
	for (int x = 0; x < 256; x++) {
		uint8_t inv = 0;
		if (x)
			for (int y = 1; y < 256; y++)
				if (gmul((uint8_t)x, (uint8_t)y) == 1) {
					inv = (uint8_t)y;
					break;
				}
		uint8_t s = inv, r = inv;
		for (int k = 0; k < 4; k++) {
			r = (uint8_t)((r << 1) | (r >> 7));
			s ^= r;
		}
		g_sbox[x] = s ^ 0x63;
	}
	g_sbox_ready = true;
}
struct AesKey {
	int rounds;
	uint8_t rk[15][16];
};
void aes_expand(const uint8_t *key, int key_bytes, AesKey &k) {
	make_sbox();
	const int nk = key_bytes / 4;
	k.rounds = nk + 6;
	uint8_t w[60][4];
	for (int i = 0; i < nk; i++) memcpy(w[i], key + 4 * i, 4);
	uint8_t rcon = 1;
	for (int i = nk; i < 4 * (k.rounds + 1); i++) {
		uint8_t t[4];
		memcpy(t, w[i - 1], 4);
		if (i % nk == 0) {
			const uint8_t t0 = t[0];
			t[0] = g_sbox[t[1]] ^ rcon;
			t[1] = g_sbox[t[2]];
			t[2] = g_sbox[t[3]];
			t[3] = g_sbox[t0];
			rcon = gmul(rcon, 2);
		} else if (nk > 6 && i % nk == 4) {
			for (int j = 0; j < 4; j++) t[j] = g_sbox[t[j]];
		}
		for (int j = 0; j < 4; j++) w[i][j] = w[i - nk][j] ^ t[j];
	}
	for (int r = 0; r <= k.rounds; r++)
		for (int c = 0; c < 4; c++) memcpy(&k.rk[r][4 * c], w[4 * r + c], 4);
}
void aes_encrypt_block(const AesKey &k, const uint8_t in[16], uint8_t out[16]) {
	uint8_t s[16];
	for (int i = 0; i < 16; i++) s[i] = in[i] ^ k.rk[0][i];
	for (int r = 1; r <= k.rounds; r++) {
		uint8_t t[16];
		for (int c = 0; c < 4; c++)
			for (int row = 0; row < 4; row++) t[4 * c + row] = g_sbox[s[4 * ((c + row) & 3) + row]]; // SubBytes + ShiftRows
		if (r < k.rounds) {
			for (int c = 0; c < 4; c++) { // MixColumns
				const uint8_t a0 = t[4 * c], a1 = t[4 * c + 1], a2 = t[4 * c + 2], a3 = t[4 * c + 3];
				s[4 * c] = gmul(a0, 2) ^ gmul(a1, 3) ^ a2 ^ a3;
				s[4 * c + 1] = a0 ^ gmul(a1, 2) ^ gmul(a2, 3) ^ a3;
				s[4 * c + 2] = a0 ^ a1 ^ gmul(a2, 2) ^ gmul(a3, 3);
				s[4 * c + 3] = gmul(a0, 3) ^ a1 ^ a2 ^ gmul(a3, 2);
			}
		} else {
			memcpy(s, t, 16);
		}
		for (int i = 0; i < 16; i++) s[i] ^= k.rk[r][i];
	}
	memcpy(out, s, 16);
}

// ---- SHA-1 (FIPS 180-4), HMAC (RFC 2104), PBKDF2 (RFC 2898) ------------------------------------------------
struct Sha1 {
	uint32_t h[5];
	uint8_t buf[64];
	uint64_t total;
	Sha1() { reset(); }
	void reset() {
		h[0] = 0x67452301u;
		h[1] = 0xEFCDAB89u;
		h[2] = 0x98BADCFEu;
		h[3] = 0x10325476u;
		h[4] = 0xC3D2E1F0u;
		total = 0;
	}
	static uint32_t rol(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }
	void block(const uint8_t *p) {
		uint32_t w[80];
		for (int i = 0; i < 16; i++) w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | p[4 * i + 3];
		for (int i = 16; i < 80; i++) w[i] = rol(w[i - 3] ^ w[i - 8] ^ w[i - 14] ^ w[i - 16], 1);
		uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
		for (int i = 0; i < 80; i++) {
			uint32_t f, k;
			if (i < 20) {
				f = (b & c) | (~b & d);
				k = 0x5A827999u;
			} else if (i < 40) {
				f = b ^ c ^ d;
				k = 0x6ED9EBA1u;
			} else if (i < 60) {
				f = (b & c) | (b & d) | (c & d);
				k = 0x8F1BBCDCu;
			} else {
				f = b ^ c ^ d;
				k = 0xCA62C1D6u;
			}
			const uint32_t t = rol(a, 5) + f + e + k + w[i];
			e = d;
			d = c;
			c = rol(b, 30);
			b = a;
			a = t;
		}
		h[0] += a;
		h[1] += b;
		h[2] += c;
		h[3] += d;
		h[4] += e;
	}
	void update(const uint8_t *p, size_t n) {
		while (n) {
			const size_t fill = (size_t)(total & 63);
			const size_t take = n < 64 - fill ? n : 64 - fill;
			memcpy(buf + fill, p, take);
			total += take;
			p += take;
			n -= take;
			if ((total & 63) == 0) block(buf);
		}
	}
	void final(uint8_t out[20]) {
		const uint64_t bits = total * 8;
		const uint8_t one = 0x80, zero = 0;
		update(&one, 1);
		while ((total & 63) != 56) update(&zero, 1);
		uint8_t len[8];
		for (int i = 0; i < 8; i++) len[i] = (uint8_t)(bits >> (56 - 8 * i));
		update(len, 8);
		for (int i = 0; i < 5; i++)
			for (int j = 0; j < 4; j++) out[4 * i + j] = (uint8_t)(h[i] >> (24 - 8 * j));
	}
};
struct Hmac {
	Sha1 inner, outer;
	void init(const uint8_t *key, size_t n) {
		uint8_t k[64] = {0};
		if (n > 64) {
			Sha1 s;
			s.update(key, n);
			s.final(k);
		} else {
			memcpy(k, key, n);
		}
		uint8_t pad[64];
		for (int i = 0; i < 64; i++) pad[i] = k[i] ^ 0x36;
		inner.reset();
		inner.update(pad, 64);
		for (int i = 0; i < 64; i++) pad[i] = k[i] ^ 0x5C;
		outer.reset();
		outer.update(pad, 64);
	}
	void update(const uint8_t *p, size_t n) { inner.update(p, n); }
	void final(uint8_t out[20]) {
		uint8_t ih[20];
		Sha1 i2 = inner, o2 = outer;
		i2.final(ih);
		o2.update(ih, 20);
		o2.final(out);
	}
};
void pbkdf2(const uint8_t *pw, size_t pwn, const uint8_t *salt, size_t sn, int rounds, uint8_t *out, size_t outn) {
	Hmac base;
	base.init(pw, pwn);
	for (uint32_t blk = 1; outn; blk++) {
		uint8_t u[20], t[20];
		Hmac h = base;
		h.update(salt, sn);
		const uint8_t be[4] = {(uint8_t)(blk >> 24), (uint8_t)(blk >> 16), (uint8_t)(blk >> 8), (uint8_t)blk};
		h.update(be, 4);
		h.final(u);
		memcpy(t, u, 20);
		for (int r = 1; r < rounds; r++) {
			Hmac g = base;
			g.update(u, 20);
			g.final(u);
			for (int i = 0; i < 20; i++) t[i] ^= u[i];
		}
		const size_t take = outn < 20 ? outn : 20;
		memcpy(out, t, take);
		out += take;
		outn -= take;
	}
}

// ---- ZipAESTransform ------------------------------------------------------------------------------------
struct AesTransform {
	int blockSize;
	AesKey enc;
	uint8_t counterNonce[32];
	uint8_t encryptBuffer[32];
	int encrPos;
	uint8_t pwdVerifier[2];
	Hmac hmac;
	bool writeMode;
	// :41-72
	AesTransform(const uint8_t *pw, size_t pwn, const uint8_t *salt, int blockSize_, bool writeMode_) : blockSize(blockSize_), writeMode(writeMode_) {
		memset(counterNonce, 0, sizeof counterNonce);
		encrPos = 16; // ENCRYPT_BLOCK
		uint8_t kb[32 + 32 + 2];
		pbkdf2(pw, pwn, salt, (size_t)blockSize / 2, 1000, kb, (size_t)(2 * blockSize + 2));
		aes_expand(kb, blockSize, enc);
		hmac.init(kb + blockSize, (size_t)blockSize);
		memcpy(pwdVerifier, kb + 2 * blockSize, 2);
	}
	// :75-112
	void TransformBlock(const uint8_t *in, size_t n, uint8_t *out) {
		if (!writeMode) hmac.update(in, n);
		for (size_t ix = 0; ix < n; ix++) {
			if (encrPos == 16) {
				int j = 0;
				while (++counterNonce[j] == 0) ++j; // little-endian increment (:91-95)
				// ECB over _blockSize bytes; only the first 16 are used (:18-21, :97)
				aes_encrypt_block(enc, counterNonce, encryptBuffer);
				encrPos = 0;
			}
			out[ix] = (uint8_t)(in[ix] ^ encryptBuffer[encrPos++]);
		}
		if (writeMode) hmac.update(out, n);
	}
};

// ---- PkzipClassic ---------------------------------------------------------------------------------------
uint32_t g_crc_table[256];
bool g_crc_ready = false;
void make_crc() {
	if (g_crc_ready) return;
	for (uint32_t i = 0; i < 256; i++) {
		uint32_t c = i;
		for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
		g_crc_table[i] = c;
	}
	g_crc_ready = true;
}
// Checksum/Crc32.cs ComputeCrc32(oldCrc, bval)
uint32_t crc_step(uint32_t old, uint8_t b) {
	make_crc();
	return g_crc_table[(old ^ b) & 0xFF] ^ (old >> 8);
}
struct Classic {
	uint32_t keys[3];
	uint8_t TransformByte() const { // :74-78
		const uint32_t temp = (keys[2] & 0xFFFF) | 2;
		return (uint8_t)((temp * (temp ^ 1)) >> 8);
	}
	void UpdateKeys(uint8_t ch) { // :105-111
		keys[0] = crc_step(keys[0], ch);
		keys[1] = keys[1] + (uint8_t)keys[0];
		keys[1] = keys[1] * 134775813u + 1u;
		keys[2] = crc_step(keys[2], (uint8_t)(keys[1] >> 24));
	}
};

} // namespace

extern "C" {

void szl_aes_encrypt_block(const uint8_t *key, int key_bytes, const uint8_t *in16, uint8_t *out16) {
	AesKey k;
	aes_expand(key, key_bytes, k);
	aes_encrypt_block(k, in16, out16);
}
void szl_sha1(const uint8_t *p, uint64_t n, uint8_t *out20) {
	Sha1 s;
	s.update(p, (size_t)n);
	s.final(out20);
}
void szl_hmac_sha1(const uint8_t *key, uint64_t kn, const uint8_t *p, uint64_t n, uint8_t *out20) {
	Hmac h;
	h.init(key, (size_t)kn);
	h.update(p, (size_t)n);
	h.final(out20);
}
void szl_pbkdf2_sha1(const uint8_t *pw, uint64_t pwn, const uint8_t *salt, uint64_t sn, int rounds, uint8_t *out, uint64_t outn) {
	pbkdf2(pw, (size_t)pwn, salt, (size_t)sn, rounds, out, (size_t)outn);
}
// new ZipAESTransform(password, salt, blockSize, writeMode); TransformBlock over `n` bytes in pieces of `piece` (0: one call);
// verifier2 <- PwdVerifier, auth20 <- GetAuthCode()
void szl_zip_aes(const uint8_t *pw, uint64_t pwn, const uint8_t *salt, int block_size, int write_mode, const uint8_t *in, uint64_t n,
                 uint64_t piece, uint8_t *out, uint8_t *verifier2, uint8_t *auth20) {
	AesTransform t(pw, (size_t)pwn, salt, block_size, write_mode != 0);
	if (piece == 0) piece = n ? n : 1;
	for (uint64_t o = 0; o < n; o += piece) t.TransformBlock(in + o, (size_t)(n - o < piece ? n - o : piece), out + o);
	memcpy(verifier2, t.pwdVerifier, 2);
	t.hmac.final(auth20);
}
// PkzipClassic.GenerateKeys(seed) (:19-50): 12 bytes, little-endian keys[0..2]
void szl_pkzip_generate_keys(const uint8_t *seed, uint64_t n, uint8_t *keys12) {
	Classic c;
	c.keys[0] = 0x12345678u;
	c.keys[1] = 0x23456789u;
	c.keys[2] = 0x34567890u;
	for (uint64_t i = 0; i < n; i++) c.UpdateKeys(seed[i]);
	for (int k = 0; k < 3; k++)
		for (int j = 0; j < 4; j++) keys12[4 * k + j] = (uint8_t)(c.keys[k] >> (8 * j));
}
// PkzipClassicEncryptCryptoTransform / DecryptCryptoTransform .TransformBlock; keys12 in (SetKeys :84-100) and out
void szl_pkzip_transform(uint8_t *keys12, int encrypt, const uint8_t *in, uint64_t n, uint8_t *out) {
	Classic c;
	for (int k = 0; k < 3; k++)
		c.keys[k] = (uint32_t)keys12[4 * k] | ((uint32_t)keys12[4 * k + 1] << 8) | ((uint32_t)keys12[4 * k + 2] << 16) | ((uint32_t)keys12[4 * k + 3] << 24);
	for (uint64_t i = 0; i < n; i++) {
		if (encrypt) {
			const uint8_t old = in[i];
			out[i] = (uint8_t)(in[i] ^ c.TransformByte());
			c.UpdateKeys(old);
		} else {
			const uint8_t nb = (uint8_t)(in[i] ^ c.TransformByte());
			out[i] = nb;
			c.UpdateKeys(nb);
		}
	}
	for (int k = 0; k < 3; k++)
		for (int j = 0; j < 4; j++) keys12[4 * k + j] = (uint8_t)(c.keys[k] >> (8 * j));
}
}
