// b200z_crypto.cu -- SURVEY.md row f4: the two entry ciphers the reference applies to compressed bytes
// (Streams/DeflaterOutputStream.cs:227-231 EncryptBlock; paths relative to SharpZipLib's src/ICSharpCode.SharpZipLib/).
//
//   WinZip AES   Encryption/ZipAESTransform.cs: constructor :41-72 (PBKDF2-HMAC-SHA1, 1000 rounds: key1 | key2 | verifier),
//                TransformBlock :75-112 (AES-CTR, little-endian counter starting at 1; HMAC-SHA1 of the ciphertext),
//                GetAuthCode :122.
//   PKZIP classic Encryption/PkzipClassic.cs: GenerateKeys :19-50, TransformByte / UpdateKeys :74-111, TransformBlock
//                :170-178 (encrypt) and :279-288 (decrypt).
//
// What is parallel and what is not.  AES-CTR is: one thread per 16-byte keystream block, T-table rounds out of shared
// memory (k_aes_ctr; the compressed bytes are already in HBM behind the deflate plan, so encrypting them costs one more
// pass over C bytes).  SHA-1 (the HMAC) and the classic cipher are serial chains per stream by construction (each 64-byte
// block / each byte depends on the one before); they run one thread per stream, i.e. they scale with the number of zip
// entries in the batch, not with the size of one entry.
#include "b200z_internal.cuh"

#include <cstring>
#include <memory>
#include <mutex>

namespace b200z {

// ---- AES tables: S-box from its definition (inverse in GF(2^8), affine map), Te0 = (2s, s, s, 3s) -----------------
__constant__ uint32_t c_te0[256];
static uint32_t h_te0[256];
static uint8_t h_sbox[256];
static std::once_flag g_tab_once;
static uint32_t h_crc[256];

static uint8_t xtime(uint8_t a) { return (uint8_t)((a << 1) ^ ((a & 0x80) ? 0x1B : 0)); }

static void build_tables() {
	// powers of the generator 3: log / antilog give the multiplicative inverse
	uint8_t alog[256], lg[256];
	uint8_t v = 1;
	for (int i = 0; i < 255; i++) {
		alog[i] = v;
		lg[v] = (uint8_t)i;
		v = (uint8_t)(v ^ xtime(v));
	}
	for (int x = 0; x < 256; x++) {
		const uint8_t inv = x ? alog[(255 - lg[x]) % 255] : 0;
		uint8_t s = inv;
		for (int k = 1; k <= 4; k++) s ^= (uint8_t)((inv << k) | (inv >> (8 - k)));
		s ^= 0x63;
		h_sbox[x] = s;
		const uint8_t s2 = xtime(s);
		h_te0[x] = ((uint32_t)s2 << 24) | ((uint32_t)s << 16) | ((uint32_t)s << 8) | (uint32_t)(s2 ^ s);
	}
	for (uint32_t i = 0; i < 256; i++) {
		uint32_t c = i;
		for (int k = 0; k < 8; k++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
		h_crc[i] = c;
	}
}

static std::mutex g_dev_mu;
static bool g_dev_ready[64];
static int crypto_ready() {
	int rc = ensure_init();
	if (rc) return rc;
	std::call_once(g_tab_once, build_tables);
	int dev = 0;
	B200Z_CUDA(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(g_dev_mu);
	if (dev >= 0 && dev < 64 && !g_dev_ready[dev]) {
		B200Z_CUDA(cudaMemcpyToSymbol(c_te0, h_te0, sizeof h_te0));
		g_dev_ready[dev] = true;
	}
	return B200Z_OK;
}

// What a stream carries from one TransformBlock to the next (zero = a fresh transform): the CTR position and the inner
// SHA-1 of the HMAC with the ciphertext bytes that do not fill a 64-byte block yet.
struct AesState {
	uint64_t bytes;
	uint32_t h[5];
	uint32_t started;
	uint8_t buf[64];
	uint8_t pad[32];
};
static_assert(sizeof(AesState) == 128, "AesState");

__device__ __forceinline__ uint32_t ror32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t rol32(uint32_t x, int n) { return __funnelshift_l(x, x, n); }
__device__ __forceinline__ uint32_t sub_word(const uint32_t *te, uint32_t w) { // S-box of every byte: S[x] = byte 2 of Te0[x]
	return (((te[w >> 24] >> 8) & 0xFFu) << 24) | (((te[(w >> 16) & 0xFFu] >> 8) & 0xFFu) << 16) |
	       (((te[(w >> 8) & 0xFFu] >> 8) & 0xFFu) << 8) | ((te[w & 0xFFu] >> 8) & 0xFFu);
}

constexpr int kAesThreads = 256;
constexpr int kAesBlocksPerThread = 4;
constexpr int kAesTile = kAesThreads * kAesBlocksPerThread * 16; // bytes of keystream per CTA and grid step
constexpr int kAesMaxTiles = 1024;                                 // CTAs per stream; longer streams loop (16 MiB per step)

// grid (streams, tiles): streams on x (up to 2^31 - 1 of them), at most kAesMaxTiles tiles on y.  keys: per stream
// 2 * key_bytes + 2 bytes (key1 | key2 | verifier).
__global__ void __launch_bounds__(kAesThreads)
    k_aes_ctr(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, const int64_t *__restrict__ off,
              const int64_t *__restrict__ len, const uint8_t *__restrict__ keys, int key_bytes, const AesState *__restrict__ state,
              int hashed) {
	__shared__ uint32_t s_te[256];
	__shared__ uint32_t s_rk[60];
	const int stream = blockIdx.x;
	const int64_t n = len[stream];
	// stream position of this call's first byte: the state's count, which the HMAC kernel has already advanced when it ran first
	const uint64_t start = state[stream].bytes - (hashed ? (uint64_t)(n > 0 ? n : 0) : 0u);
	const uint64_t first_blk = start >> 4, last_blk = (start + (uint64_t)n + 15) >> 4;
	if (n <= 0 || first_blk + (uint64_t)blockIdx.y * (kAesTile / 16) >= last_blk) return;
	s_te[threadIdx.x] = c_te0[threadIdx.x];
	__syncthreads();
	const int nk = key_bytes / 4, rounds = nk + 6;
	if (threadIdx.x == 0) {
		// key schedule (FIPS 197 5.2) on big-endian words
		const uint8_t *k = keys + (int64_t)stream * (2 * key_bytes + 2);
		for (int i = 0; i < nk; i++)
			s_rk[i] = ((uint32_t)k[4 * i] << 24) | ((uint32_t)k[4 * i + 1] << 16) | ((uint32_t)k[4 * i + 2] << 8) | k[4 * i + 3];
		uint32_t rcon = 1;
		for (int i = nk; i < 4 * (rounds + 1); i++) {
			uint32_t t = s_rk[i - 1];
			if (i % nk == 0) {
				t = sub_word(s_te, rol32(t, 8)) ^ (rcon << 24);
				rcon = (rcon << 1) ^ ((rcon & 0x80u) ? 0x11Bu : 0u);
			} else if (nk > 6 && i % nk == 4) {
				t = sub_word(s_te, t);
			}
			s_rk[i] = s_rk[i - nk] ^ t;
		}
	}
	__syncthreads();
	const uint8_t *src = in + off[stream];
	uint8_t *dst = out + off[stream];
	for (uint64_t tb = first_blk + (uint64_t)blockIdx.y * (kAesTile / 16); tb < last_blk; tb += (uint64_t)gridDim.y * (kAesTile / 16)) {
#pragma unroll
		for (int j = 0; j < kAesBlocksPerThread; j++) {
			const uint64_t kb = tb + (uint64_t)j * kAesThreads + threadIdx.x;
			if (kb >= last_blk) break;
			// the nonce is a little-endian counter that starts at 1 (:88-95); the block's bytes 0..3 as a big-endian word
			const uint64_t ctr = kb + 1;
			uint32_t s0 = __byte_perm((uint32_t)ctr, 0, 0x0123) ^ s_rk[0];
			uint32_t s1 = __byte_perm((uint32_t)(ctr >> 32), 0, 0x0123) ^ s_rk[1];
			uint32_t s2 = s_rk[2], s3 = s_rk[3];
			for (int r = 1; r < rounds; r++) {
				const uint32_t t0 = s_te[s0 >> 24] ^ ror32(s_te[(s1 >> 16) & 0xFFu], 8) ^ ror32(s_te[(s2 >> 8) & 0xFFu], 16) ^
				                    ror32(s_te[s3 & 0xFFu], 24) ^ s_rk[4 * r];
				const uint32_t t1 = s_te[s1 >> 24] ^ ror32(s_te[(s2 >> 16) & 0xFFu], 8) ^ ror32(s_te[(s3 >> 8) & 0xFFu], 16) ^
				                    ror32(s_te[s0 & 0xFFu], 24) ^ s_rk[4 * r + 1];
				const uint32_t t2 = s_te[s2 >> 24] ^ ror32(s_te[(s3 >> 16) & 0xFFu], 8) ^ ror32(s_te[(s0 >> 8) & 0xFFu], 16) ^
				                    ror32(s_te[s1 & 0xFFu], 24) ^ s_rk[4 * r + 2];
				const uint32_t t3 = s_te[s3 >> 24] ^ ror32(s_te[(s0 >> 16) & 0xFFu], 8) ^ ror32(s_te[(s1 >> 8) & 0xFFu], 16) ^
				                    ror32(s_te[s2 & 0xFFu], 24) ^ s_rk[4 * r + 3];
				s0 = t0;
				s1 = t1;
				s2 = t2;
				s3 = t3;
			}
#define B200Z_SB(x) ((s_te[(x)] >> 8) & 0xFFu)
			uint32_t k0 = (B200Z_SB(s0 >> 24) << 24) | (B200Z_SB((s1 >> 16) & 0xFFu) << 16) | (B200Z_SB((s2 >> 8) & 0xFFu) << 8) | B200Z_SB(s3 & 0xFFu);
			uint32_t k1 = (B200Z_SB(s1 >> 24) << 24) | (B200Z_SB((s2 >> 16) & 0xFFu) << 16) | (B200Z_SB((s3 >> 8) & 0xFFu) << 8) | B200Z_SB(s0 & 0xFFu);
			uint32_t k2 = (B200Z_SB(s2 >> 24) << 24) | (B200Z_SB((s3 >> 16) & 0xFFu) << 16) | (B200Z_SB((s0 >> 8) & 0xFFu) << 8) | B200Z_SB(s1 & 0xFFu);
			uint32_t k3 = (B200Z_SB(s3 >> 24) << 24) | (B200Z_SB((s0 >> 16) & 0xFFu) << 16) | (B200Z_SB((s1 >> 8) & 0xFFu) << 8) | B200Z_SB(s2 & 0xFFu);
#undef B200Z_SB
			// keystream bytes in memory order
			k0 = __byte_perm(k0 ^ s_rk[4 * rounds], 0, 0x0123);
			k1 = __byte_perm(k1 ^ s_rk[4 * rounds + 1], 0, 0x0123);
			k2 = __byte_perm(k2 ^ s_rk[4 * rounds + 2], 0, 0x0123);
			k3 = __byte_perm(k3 ^ s_rk[4 * rounds + 3], 0, 0x0123);
			const int64_t i0 = (int64_t)(kb * 16) - (int64_t)start; // data index of the block's first byte
			if (i0 >= 0 && i0 + 16 <= n && (((uintptr_t)(src + i0) | (uintptr_t)(dst + i0)) & 15u) == 0) {
				uint4 d = *reinterpret_cast<const uint4 *>(src + i0);
				d.x ^= k0;
				d.y ^= k1;
				d.z ^= k2;
				d.w ^= k3;
				*reinterpret_cast<uint4 *>(dst + i0) = d;
			} else {
				const uint32_t kk[4] = {k0, k1, k2, k3};
#pragma unroll
				for (int b = 0; b < 16; b++) {
					const int64_t i = i0 + b;
					if (i >= 0 && i < n) dst[i] = (uint8_t)(src[i] ^ (uint8_t)(kk[b >> 2] >> (8 * (b & 3))));
				}
			}
		}
	}
}

// ---- SHA-1 --------------------------------------------------------------------------------------------------------
struct Sha1Regs {
	uint32_t h[5];
};
__device__ __forceinline__ void sha1_init(Sha1Regs &s) {
	s.h[0] = 0x67452301u;
	s.h[1] = 0xEFCDAB89u;
	s.h[2] = 0x98BADCFEu;
	s.h[3] = 0x10325476u;
	s.h[4] = 0xC3D2E1F0u;
}
// one 64-byte block given as 16 big-endian words (FIPS 180-4 6.1.2, the 16-word circular schedule)
__device__ __forceinline__ void sha1_block(Sha1Regs &s, uint32_t w[16]) {
	uint32_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4];
#pragma unroll
	for (int i = 0; i < 80; i++) {
		uint32_t wi;
		if (i < 16) wi = w[i];
		else {
			wi = rol32(w[(i + 13) & 15] ^ w[(i + 8) & 15] ^ w[(i + 2) & 15] ^ w[i & 15], 1);
			w[i & 15] = wi;
		}
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
		const uint32_t t = rol32(a, 5) + f + e + k + wi;
		e = d;
		d = c;
		c = rol32(b, 30);
		b = a;
		a = t;
	}
	s.h[0] += a;
	s.h[1] += b;
	s.h[2] += c;
	s.h[3] += d;
	s.h[4] += e;
}
// key (<= 64 bytes) xor pad as one block
__device__ __forceinline__ void sha1_key_block(Sha1Regs &s, const uint8_t *key, int kn, uint32_t pad) {
	uint32_t w[16];
#pragma unroll
	for (int i = 0; i < 16; i++) {
		uint32_t v = 0;
		for (int j = 0; j < 4; j++) v = (v << 8) | (uint32_t)(4 * i + j < kn ? key[4 * i + j] : 0);
		w[i] = v ^ pad;
	}
	sha1_block(s, w);
}
// a message of 20 bytes (five words) behind a 64-byte key block: one padded block, total 84 bytes
__device__ __forceinline__ void sha1_digest_block(Sha1Regs &s, const uint32_t m[5]) {
	uint32_t w[16];
#pragma unroll
	for (int i = 0; i < 5; i++) w[i] = m[i];
	w[5] = 0x80000000u;
#pragma unroll
	for (int i = 6; i < 15; i++) w[i] = 0;
	w[15] = (64 + 20) * 8;
	sha1_block(s, w);
}

// One thread per stream: the HMAC's inner hash runs over this call's ciphertext; with `finish` the 20-byte code is written.
__global__ void __launch_bounds__(64)
    k_hmac_sha1(const uint8_t *__restrict__ ct, const int64_t *__restrict__ off, const int64_t *__restrict__ len,
                const uint8_t *__restrict__ keys, int key_bytes, AesState *__restrict__ state, int finish, uint8_t *__restrict__ auth,
                int n) {
	const int stream = blockIdx.x * blockDim.x + threadIdx.x;
	if (stream >= n) return;
	AesState &st = state[stream];
	const uint8_t *key2 = keys + (int64_t)stream * (2 * key_bytes + 2) + key_bytes;
	Sha1Regs s;
	if (!st.started) {
		sha1_init(s);
		sha1_key_block(s, key2, key_bytes, 0x36363636u);
	} else {
#pragma unroll
		for (int i = 0; i < 5; i++) s.h[i] = st.h[i];
	}
	const uint8_t *p = ct + off[stream];
	int64_t m = len[stream] > 0 ? len[stream] : 0;
	uint32_t fill = (uint32_t)(st.bytes & 63u);
	uint64_t total = st.bytes;
	uint32_t w[16];
	// top up a partial block first
	if (fill) {
		while (fill < 64 && m > 0) {
			st.buf[fill++] = *p++;
			--m;
			++total;
		}
		if (fill == 64) {
#pragma unroll
			for (int i = 0; i < 16; i++)
				w[i] = ((uint32_t)st.buf[4 * i] << 24) | ((uint32_t)st.buf[4 * i + 1] << 16) | ((uint32_t)st.buf[4 * i + 2] << 8) | st.buf[4 * i + 3];
			sha1_block(s, w);
			fill = 0;
		}
	}
	if ((((uintptr_t)p) & 15u) == 0) {
		for (; m >= 64; m -= 64, p += 64, total += 64) {
#pragma unroll
			for (int q = 0; q < 4; q++) {
				const uint4 v = reinterpret_cast<const uint4 *>(p)[q];
				w[4 * q] = __byte_perm(v.x, 0, 0x0123);
				w[4 * q + 1] = __byte_perm(v.y, 0, 0x0123);
				w[4 * q + 2] = __byte_perm(v.z, 0, 0x0123);
				w[4 * q + 3] = __byte_perm(v.w, 0, 0x0123);
			}
			sha1_block(s, w);
		}
	} else {
		for (; m >= 64; m -= 64, p += 64, total += 64) {
#pragma unroll
			for (int i = 0; i < 16; i++)
				w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | p[4 * i + 3];
			sha1_block(s, w);
		}
	}
	while (m > 0) {
		st.buf[fill++] = *p++;
		--m;
		++total;
	}
	st.bytes = total;
	st.started = 1;
#pragma unroll
	for (int i = 0; i < 5; i++) st.h[i] = s.h[i];
	if (finish) {
		// inner: padding behind 64 + total bytes; outer: SHA-1((key2 ^ opad) | inner digest)  (RFC 2104)
		uint8_t last[128];
		const uint32_t f = (uint32_t)(total & 63u);
		for (uint32_t i = 0; i < f; i++) last[i] = st.buf[i];
		last[f] = 0x80;
		const uint32_t blocks = f < 56 ? 1u : 2u;
		for (uint32_t i = f + 1; i < 64 * blocks - 8; i++) last[i] = 0;
		const uint64_t bits = (64 + total) * 8;
		for (int i = 0; i < 8; i++) last[64 * blocks - 8 + i] = (uint8_t)(bits >> (56 - 8 * i));
		for (uint32_t b = 0; b < blocks; b++) {
			for (int i = 0; i < 16; i++)
				w[i] = ((uint32_t)last[64 * b + 4 * i] << 24) | ((uint32_t)last[64 * b + 4 * i + 1] << 16) |
				       ((uint32_t)last[64 * b + 4 * i + 2] << 8) | last[64 * b + 4 * i + 3];
			sha1_block(s, w);
		}
		Sha1Regs o;
		sha1_init(o);
		sha1_key_block(o, key2, key_bytes, 0x5C5C5C5Cu);
		sha1_digest_block(o, s.h);
		for (int i = 0; i < 5; i++)
			for (int j = 0; j < 4; j++) auth[20ll * stream + 4 * i + j] = (uint8_t)(o.h[i] >> (24 - 8 * j));
	}
}

// PBKDF2-HMAC-SHA1 (RFC 2898 5.2), 1000 rounds: one thread per (stream, 20-byte output block).  pw_off: n + 1 offsets into the
// password blob; salts: n x key_bytes / 2; out: n x (2 * key_bytes + 2).
__global__ void __launch_bounds__(64)
    k_pbkdf2(const uint8_t *__restrict__ pw, const int64_t *__restrict__ pw_off, const uint8_t *__restrict__ salts, int key_bytes,
             int rounds, uint8_t *__restrict__ out, int n) {
	const int nblk = (2 * key_bytes + 2 + 19) / 20;
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (int64_t)n * nblk) return;
	const int stream = (int)(t / nblk), blk = (int)(t % nblk) + 1;
	const uint8_t *p = pw + pw_off[stream];
	const int pn = (int)(pw_off[stream + 1] - pw_off[stream]);
	uint8_t kbuf[64];
	int kn = pn;
	if (pn > 64) { // keys longer than a block are hashed first (RFC 2104)
		Sha1Regs hk;
		sha1_init(hk);
		uint32_t w[16];
		int done = 0;
		for (; done + 64 <= pn; done += 64) {
			for (int i = 0; i < 16; i++)
				w[i] = ((uint32_t)p[done + 4 * i] << 24) | ((uint32_t)p[done + 4 * i + 1] << 16) | ((uint32_t)p[done + 4 * i + 2] << 8) | p[done + 4 * i + 3];
			sha1_block(hk, w);
		}
		uint8_t last[128];
		const int f = pn - done;
		for (int i = 0; i < f; i++) last[i] = p[done + i];
		last[f] = 0x80;
		const int blocks = f < 56 ? 1 : 2;
		for (int i = f + 1; i < 64 * blocks - 8; i++) last[i] = 0;
		const uint64_t bits = (uint64_t)pn * 8;
		for (int i = 0; i < 8; i++) last[64 * blocks - 8 + i] = (uint8_t)(bits >> (56 - 8 * i));
		for (int b = 0; b < blocks; b++) {
			for (int i = 0; i < 16; i++)
				w[i] = ((uint32_t)last[64 * b + 4 * i] << 24) | ((uint32_t)last[64 * b + 4 * i + 1] << 16) |
				       ((uint32_t)last[64 * b + 4 * i + 2] << 8) | last[64 * b + 4 * i + 3];
			sha1_block(hk, w);
		}
		for (int i = 0; i < 5; i++)
			for (int j = 0; j < 4; j++) kbuf[4 * i + j] = (uint8_t)(hk.h[i] >> (24 - 8 * j));
		kn = 20;
	} else {
		for (int i = 0; i < pn; i++) kbuf[i] = p[i];
	}
	Sha1Regs ipad, opad;
	sha1_init(ipad);
	sha1_key_block(ipad, kbuf, kn, 0x36363636u);
	sha1_init(opad);
	sha1_key_block(opad, kbuf, kn, 0x5C5C5C5Cu);
	// U1 = HMAC(pw, salt | INT(blk))
	const int sn = key_bytes / 2;
	uint32_t u[5], acc[5];
	{
		uint8_t m[64];
		for (int i = 0; i < sn; i++) m[i] = salts[(int64_t)stream * sn + i];
		m[sn] = 0;
		m[sn + 1] = 0;
		m[sn + 2] = 0;
		m[sn + 3] = (uint8_t)blk;
		const int ml = sn + 4;
		m[ml] = 0x80;
		for (int i = ml + 1; i < 56; i++) m[i] = 0;
		const uint64_t bits = (uint64_t)(64 + ml) * 8;
		for (int i = 0; i < 8; i++) m[56 + i] = (uint8_t)(bits >> (56 - 8 * i));
		uint32_t w[16];
		for (int i = 0; i < 16; i++) w[i] = ((uint32_t)m[4 * i] << 24) | ((uint32_t)m[4 * i + 1] << 16) | ((uint32_t)m[4 * i + 2] << 8) | m[4 * i + 3];
		Sha1Regs a = ipad;
		sha1_block(a, w);
		Sha1Regs b = opad;
		sha1_digest_block(b, a.h);
		for (int i = 0; i < 5; i++) u[i] = acc[i] = b.h[i];
	}
	for (int r = 1; r < rounds; r++) {
		Sha1Regs a = ipad;
		sha1_digest_block(a, u);
		Sha1Regs b = opad;
		sha1_digest_block(b, a.h);
#pragma unroll
		for (int i = 0; i < 5; i++) {
			u[i] = b.h[i];
			acc[i] ^= u[i];
		}
	}
	const int total = 2 * key_bytes + 2;
	for (int i = 0; i < 20; i++) {
		const int o = 20 * (blk - 1) + i;
		if (o < total) out[(int64_t)stream * total + o] = (uint8_t)(acc[i >> 2] >> (24 - 8 * (i & 3)));
	}
}

// ---- PKZIP classic: one thread per stream, keys[3] in and out ------------------------------------------------------
__global__ void __launch_bounds__(64)
    k_pkzip(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, const int64_t *__restrict__ off,
            const int64_t *__restrict__ len, uint32_t *__restrict__ keys, const uint32_t *__restrict__ crc_tab, int encrypt, int n) {
	__shared__ uint32_t s_crc[256];
	for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = crc_tab[i];
	__syncthreads();
	const int stream = blockIdx.x * blockDim.x + threadIdx.x;
	if (stream >= n) return;
	uint32_t k0 = keys[3 * stream], k1 = keys[3 * stream + 1], k2 = keys[3 * stream + 2];
	const uint8_t *p = in + off[stream];
	uint8_t *q = out + off[stream];
	const int64_t m = len[stream];
	for (int64_t i = 0; i < m; i++) {
		const uint32_t temp = (k2 & 0xFFFFu) | 2u; // TransformByte :74-78
		const uint8_t ks = (uint8_t)((temp * (temp ^ 1u)) >> 8);
		const uint8_t c = p[i];
		const uint8_t o = (uint8_t)(c ^ ks);
		q[i] = o;
		const uint8_t plain = encrypt ? c : o; // UpdateKeys takes the plaintext byte (:172-176, :284-286)
		k0 = s_crc[(k0 ^ plain) & 0xFFu] ^ (k0 >> 8);
		k1 = (k1 + (k0 & 0xFFu)) * 134775813u + 1u;
		k2 = s_crc[(k2 ^ (k1 >> 24)) & 0xFFu] ^ (k2 >> 8);
	}
	keys[3 * stream] = k0;
	keys[3 * stream + 1] = k1;
	keys[3 * stream + 2] = k2;
}

static int check_key_bytes(int key_bytes) {
	if (key_bytes != 16 && key_bytes != 32) { // ZipAESTransform.cs:43-44
		set_error("Invalid blocksize %d. Must be 16 or 32.", key_bytes);
		return B200Z_E_ARG;
	}
	return B200Z_OK;
}

// reading: HMAC of the input, then CTR (:79-100); writing: CTR, then HMAC of the output (:84-109).  In place is fine either way.
static int aes_launch(const uint8_t *d_in, uint8_t *d_out, const int64_t *d_off, const int64_t *d_len, int64_t max_len, int n,
                      int key_bytes, const uint8_t *d_keys, int write_mode, AesState *d_state, int finish, uint8_t *d_auth,
                      cudaStream_t s) {
	if (n <= 0) return B200Z_OK;
	int64_t tiles = (max_len + 16 + kAesTile - 1) / kAesTile;
	if (tiles < 1) tiles = 1;
	if (tiles > kAesMaxTiles) tiles = kAesMaxTiles;
	// any int32 stream count fits gridDim.x and the tiles fit gridDim.y, so neither launch can be refused for its shape after
	// the other one has run and advanced the carried state
	const dim3 grid((unsigned)n, (unsigned)tiles);
	const int hb = (n + 63) / 64;
	if (write_mode) {
		k_aes_ctr<<<grid, kAesThreads, 0, s>>>(d_in, d_out, d_off, d_len, d_keys, key_bytes, d_state, 0);
		k_hmac_sha1<<<hb, 64, 0, s>>>(d_out, d_off, d_len, d_keys, key_bytes, d_state, finish, d_auth, n);
	} else {
		k_hmac_sha1<<<hb, 64, 0, s>>>(d_in, d_off, d_len, d_keys, key_bytes, d_state, finish, d_auth, n);
		k_aes_ctr<<<grid, kAesThreads, 0, s>>>(d_in, d_out, d_off, d_len, d_keys, key_bytes, d_state, 1);
	}
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

} // namespace b200z

using namespace b200z;

struct b200z_aes_transform {
	int device = -1, key_bytes = 16, write_mode = 0;
	uint8_t keys[66];
	DevBuf d_keys, d_state, d_auth, d_meta; // d_meta: off, len
	DevBuf d_buf;                           // input in the first half, output in the second
	bool have_auth = false;
	uint8_t auth[20];
};

extern "C" {

int64_t b200z_aes_state_bytes(void) { return (int64_t)sizeof(AesState); }

int b200z_aes_derive_keys(const uint8_t *passwords, const int64_t *pw_off, const uint8_t *salts, int32_t key_bytes, int32_t n,
                          uint8_t *keys_out) {
	int rc = check_key_bytes(key_bytes);
	if (rc) return rc;
	if (n < 0 || (n > 0 && (!pw_off || !salts || !keys_out))) {
		set_error("b200z_aes_derive_keys: null argument");
		return B200Z_E_ARG;
	}
	if (n == 0) return B200Z_OK;
	rc = crypto_ready();
	if (rc) return rc;
	const int64_t pwn = pw_off[n], sn = (int64_t)n * key_bytes / 2, on = (int64_t)n * (2 * key_bytes + 2);
	Arena lay; // offsets only: the blob is `d`
	const Slot<uint8_t> o_pw = lay.reserve<uint8_t>(pwn + 16), o_salt = lay.reserve<uint8_t>(sn), o_out = lay.reserve<uint8_t>(on);
	const Slot<int64_t> o_off = lay.reserve<int64_t>(n + 1);
	DevBuf d;
	if ((rc = d.ensure((size_t)lay.used))) return rc;
	uint8_t *d_pw = d.at(o_pw), *d_salt = d.at(o_salt), *d_out = d.at(o_out);
	int64_t *d_off = d.at(o_off);
	if (pwn) B200Z_CUDA(cudaMemcpy(d_pw, passwords, (size_t)pwn, cudaMemcpyHostToDevice));
	B200Z_CUDA(cudaMemcpy(d_off, pw_off, 8ull * (n + 1), cudaMemcpyHostToDevice));
	B200Z_CUDA(cudaMemcpy(d_salt, salts, (size_t)sn, cudaMemcpyHostToDevice));
	const int nblk = (2 * key_bytes + 2 + 19) / 20;
	k_pbkdf2<<<(unsigned)(((int64_t)n * nblk + 63) / 64), 64, 0, 0>>>(d_pw, d_off, d_salt, key_bytes, 1000, d_out, n);
	B200Z_CUDA(cudaGetLastError());
	B200Z_CUDA(cudaMemcpy(keys_out, d_out, (size_t)on, cudaMemcpyDeviceToHost));
	return B200Z_OK;
}

int b200z_aes_device(const uint8_t *d_in, uint8_t *d_out, const int64_t *d_off, const int64_t *d_len, int64_t max_len, int32_t n,
                     int32_t key_bytes, const uint8_t *d_keys, int32_t write_mode, uint8_t *d_state, int32_t finish,
                     uint8_t *d_auth, void *cuda_stream) {
	int rc = check_key_bytes(key_bytes);
	if (rc) return rc;
	if (n < 0 || (n > 0 && (!d_in || !d_out || !d_off || !d_len || !d_keys || !d_state)) || (finish && n > 0 && !d_auth)) {
		set_error("b200z_aes_device: null argument");
		return B200Z_E_ARG;
	}
	rc = crypto_ready();
	if (rc) return rc;
	return aes_launch(d_in, d_out, d_off, d_len, max_len, n, key_bytes, d_keys, write_mode ? 1 : 0, reinterpret_cast<AesState *>(d_state), finish, d_auth,
	                  (cudaStream_t)cuda_stream);
}

int b200z_aes_batch(const uint8_t *const *in, const int64_t *len, int32_t n, int32_t key_bytes, const uint8_t *keys, int32_t write_mode,
                    uint8_t *const *out, uint8_t *auth) {
	int rc = check_key_bytes(key_bytes);
	if (rc) return rc;
	if (n < 0 || (n > 0 && (!in || !len || !keys || !out || !auth))) {
		set_error("b200z_aes_batch: null argument");
		return B200Z_E_ARG;
	}
	if (n == 0) return B200Z_OK;
	rc = crypto_ready();
	if (rc) return rc;
	std::vector<int64_t> off(n);
	int64_t total = 0, max_len = 0;
	for (int i = 0; i < n; i++) {
		if (len[i] < 0) {
			set_error("b200z_aes_batch: negative length");
			return B200Z_E_ARG;
		}
		off[i] = total;
		total += align_up(len[i], 256);
		max_len = std::max(max_len, len[i]);
	}
	const int64_t kb = (int64_t)n * (2 * key_bytes + 2);
	Arena lay; // offsets only: the blob is `d`
	const Slot<uint8_t> o_in = lay.reserve<uint8_t>(total + 256), o_out = lay.reserve<uint8_t>(total + 256);
	const Slot<int64_t> o_off = lay.reserve<int64_t>(n), o_len = lay.reserve<int64_t>(n);
	const Slot<uint8_t> o_keys = lay.reserve<uint8_t>(kb), o_state = lay.reserve<uint8_t>(128ll * n), o_auth = lay.reserve<uint8_t>(20ll * n);
	DevBuf d;
	if ((rc = d.ensure((size_t)lay.used))) return rc;
	B200Z_CUDA(cudaMemset(d.at(o_state), 0, 128ull * n));
	for (int i = 0; i < n; i++)
		if (len[i]) B200Z_CUDA(cudaMemcpyAsync(d.at(o_in) + off[i], in[i], (size_t)len[i], cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_off), off.data(), 8ull * n, cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_len), len, 8ull * n, cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_keys), keys, (size_t)kb, cudaMemcpyHostToDevice, 0));
	rc = b200z_aes_device(d.at(o_in), d.at(o_out), d.at(o_off), d.at(o_len), max_len, n, key_bytes, d.at(o_keys), write_mode, d.at(o_state), 1,
	                      d.at(o_auth), nullptr);
	if (rc) return rc;
	for (int i = 0; i < n; i++)
		if (len[i]) B200Z_CUDA(cudaMemcpyAsync(out[i], d.at(o_out) + off[i], (size_t)len[i], cudaMemcpyDeviceToHost, 0));
	B200Z_CUDA(cudaMemcpyAsync(auth, d.at(o_auth), 20ull * n, cudaMemcpyDeviceToHost, 0));
	B200Z_CUDA(cudaStreamSynchronize(0));
	return B200Z_OK;
}

// ---- new ZipAESTransform(key, saltBytes, blockSize, writeMode) as a handle ---------------------------------------------
int b200z_aes_transform_create(const uint8_t *password, int32_t password_len, const uint8_t *salt, int32_t key_bytes, int32_t write_mode,
                               b200z_aes_transform **out) {
	if (!out || !salt || password_len < 0 || (password_len > 0 && !password)) {
		set_error("b200z_aes_transform_create: null argument");
		return B200Z_E_ARG;
	}
	*out = nullptr;
	int rc = check_key_bytes(key_bytes);
	if (rc) return rc;
	std::unique_ptr<b200z_aes_transform> t(new b200z_aes_transform());
	t->key_bytes = key_bytes;
	t->write_mode = write_mode ? 1 : 0;
	const int64_t pw_off[2] = {0, password_len};
	rc = b200z_aes_derive_keys(password, pw_off, salt, key_bytes, 1, t->keys);
	if (rc) return rc;
	t->device = current_device();
	if ((rc = t->d_keys.ensure(256)) || (rc = t->d_state.ensure(128)) || (rc = t->d_auth.ensure(32)) || (rc = t->d_meta.ensure(16)) ||
	    (rc = t->d_buf.ensure(2 << 16)))
		return rc;
	B200Z_CUDA(cudaMemset(t->d_state.p, 0, 128));
	B200Z_CUDA(cudaMemcpy(t->d_keys.p, t->keys, (size_t)(2 * key_bytes + 2), cudaMemcpyHostToDevice));
	*out = t.release();
	return B200Z_OK;
}

// TransformBlock(inputBuffer, inputOffset, inputCount, outputBuffer, outputOffset) (:75-112)
int b200z_aes_transform_block(b200z_aes_transform *t, const uint8_t *in, int64_t count, uint8_t *out) {
	if (!t || count < 0 || (count > 0 && (!in || !out))) {
		set_error("b200z_aes_transform_block: null argument");
		return B200Z_E_ARG;
	}
	if (count == 0) return B200Z_OK;
	DeviceGuard g(t->device);
	int rc = t->d_buf.ensure(2 * (size_t)align_up(count, 65536));
	if (rc) return rc;
	uint8_t *d_out = t->d_buf.p + t->d_buf.cap / 2;
	int64_t *d_meta = reinterpret_cast<int64_t *>(t->d_meta.p);
	const int64_t meta[2] = {0, count};
	B200Z_CUDA(cudaMemcpyAsync(d_meta, meta, 16, cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(t->d_buf.p, in, (size_t)count, cudaMemcpyHostToDevice, 0));
	rc = b200z_aes_device(t->d_buf.p, d_out, d_meta, d_meta + 1, count, 1, t->key_bytes, t->d_keys.p, t->write_mode, t->d_state.p, 0, nullptr,
	                      nullptr);
	if (rc) return rc;
	B200Z_CUDA(cudaMemcpyAsync(out, d_out, (size_t)count, cudaMemcpyDeviceToHost, 0));
	B200Z_CUDA(cudaStreamSynchronize(0));
	return B200Z_OK;
}

// PwdVerifier (:117)
int b200z_aes_transform_pwd_verifier(const b200z_aes_transform *t, uint8_t *out2) {
	if (!t || !out2) {
		set_error("b200z_aes_transform_pwd_verifier: null argument");
		return B200Z_E_ARG;
	}
	memcpy(out2, t->keys + 2 * t->key_bytes, 2);
	return B200Z_OK;
}

// GetAuthCode() (:122): the HMAC of everything transformed so far, computed once (`_authCode ?? ...`)
int b200z_aes_transform_auth_code(b200z_aes_transform *t, uint8_t *out20) {
	if (!t || !out20) {
		set_error("b200z_aes_transform_auth_code: null argument");
		return B200Z_E_ARG;
	}
	if (!t->have_auth) {
		DeviceGuard g(t->device);
		int64_t *d_meta = reinterpret_cast<int64_t *>(t->d_meta.p);
		const int64_t meta[2] = {0, 0};
		B200Z_CUDA(cudaMemcpyAsync(d_meta, meta, 16, cudaMemcpyHostToDevice, 0));
		k_hmac_sha1<<<1, 64, 0, 0>>>(t->d_buf.p, d_meta, d_meta + 1, t->d_keys.p, t->key_bytes, reinterpret_cast<AesState *>(t->d_state.p), 1, t->d_auth.p, 1);
		B200Z_CUDA(cudaGetLastError());
		B200Z_CUDA(cudaMemcpy(t->auth, t->d_auth.p, 20, cudaMemcpyDeviceToHost));
		t->have_auth = true;
	}
	memcpy(out20, t->auth, 20);
	return B200Z_OK;
}

int b200z_aes_transform_destroy(b200z_aes_transform *t) {
	if (!t) return B200Z_OK;
	DeviceGuard g(t->device);
	delete t;
	return B200Z_OK;
}

// ---- PKZIP classic -------------------------------------------------------------------------------------------------
// PkzipClassic.GenerateKeys(seed) (:19-50): key set-up from the password bytes, 3 CRC steps per byte -- host side, like the
// reference's own callers do it before they create the transform.
int b200z_pkzip_generate_keys(const uint8_t *seed, int64_t n, uint8_t *keys12) {
	if (!seed || !keys12) { // :21-24
		set_error("b200z_pkzip_generate_keys: null argument");
		return B200Z_E_ARG;
	}
	if (n == 0) { // :26-29
		set_error("Length is zero");
		return B200Z_E_ARG;
	}
	std::call_once(g_tab_once, build_tables);
	uint32_t k[3] = {0x12345678u, 0x23456789u, 0x34567890u};
	for (int64_t i = 0; i < n; i++) {
		k[0] = h_crc[(k[0] ^ seed[i]) & 0xFF] ^ (k[0] >> 8);
		k[1] = (k[1] + (k[0] & 0xFF)) * 134775813u + 1u;
		k[2] = h_crc[(k[2] ^ (k[1] >> 24)) & 0xFF] ^ (k[2] >> 8);
	}
	for (int j = 0; j < 3; j++)
		for (int b = 0; b < 4; b++) keys12[4 * j + b] = (uint8_t)(k[j] >> (8 * b));
	return B200Z_OK;
}

static int pkzip_table(const uint32_t **d_tab) {
	static std::mutex mu;
	static uint32_t *tabs[64];
	int rc = crypto_ready();
	if (rc) return rc;
	int dev = 0;
	B200Z_CUDA(cudaGetDevice(&dev));
	std::lock_guard<std::mutex> lk(mu);
	if (dev < 0 || dev >= 64) {
		set_error("device index out of range");
		return B200Z_E_ARG;
	}
	if (!tabs[dev]) {
		B200Z_CUDA(cudaMalloc(&tabs[dev], sizeof h_crc));
		B200Z_CUDA(cudaMemcpy(tabs[dev], h_crc, sizeof h_crc, cudaMemcpyHostToDevice));
	}
	*d_tab = tabs[dev];
	return B200Z_OK;
}

int b200z_pkzip_device(const uint8_t *d_in, uint8_t *d_out, const int64_t *d_off, const int64_t *d_len, int32_t n, uint32_t *d_keys,
                       int32_t encrypt, void *cuda_stream) {
	if (n < 0 || (n > 0 && (!d_in || !d_out || !d_off || !d_len || !d_keys))) {
		set_error("b200z_pkzip_device: null argument");
		return B200Z_E_ARG;
	}
	if (n == 0) return B200Z_OK;
	const uint32_t *tab = nullptr;
	int rc = pkzip_table(&tab);
	if (rc) return rc;
	k_pkzip<<<(n + 63) / 64, 64, 0, (cudaStream_t)cuda_stream>>>(d_in, d_out, d_off, d_len, d_keys, tab, encrypt ? 1 : 0, n);
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

int b200z_pkzip_batch(const uint8_t *const *in, const int64_t *len, int32_t n, uint8_t *keys12, int32_t encrypt, uint8_t *const *out) {
	if (n < 0 || (n > 0 && (!in || !len || !keys12 || !out))) {
		set_error("b200z_pkzip_batch: null argument");
		return B200Z_E_ARG;
	}
	if (n == 0) return B200Z_OK;
	int rc = crypto_ready();
	if (rc) return rc;
	std::vector<int64_t> off(n);
	int64_t total = 0;
	for (int i = 0; i < n; i++) {
		if (len[i] < 0) {
			set_error("b200z_pkzip_batch: negative length");
			return B200Z_E_ARG;
		}
		off[i] = total;
		total += align_up(len[i], 256);
	}
	std::vector<uint32_t> k(3 * (size_t)n);
	for (int i = 0; i < 3 * n; i++)
		k[i] = (uint32_t)keys12[4 * i] | ((uint32_t)keys12[4 * i + 1] << 8) | ((uint32_t)keys12[4 * i + 2] << 16) | ((uint32_t)keys12[4 * i + 3] << 24);
	Arena lay; // offsets only: the blob is `d`
	const Slot<uint8_t> o_in = lay.reserve<uint8_t>(total + 256), o_out = lay.reserve<uint8_t>(total + 256);
	const Slot<int64_t> o_off = lay.reserve<int64_t>(n), o_len = lay.reserve<int64_t>(n);
	const Slot<uint32_t> o_keys = lay.reserve<uint32_t>(3ll * n);
	DevBuf d;
	if ((rc = d.ensure((size_t)lay.used))) return rc;
	for (int i = 0; i < n; i++)
		if (len[i]) B200Z_CUDA(cudaMemcpyAsync(d.at(o_in) + off[i], in[i], (size_t)len[i], cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_off), off.data(), 8ull * n, cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_len), len, 8ull * n, cudaMemcpyHostToDevice, 0));
	B200Z_CUDA(cudaMemcpyAsync(d.at(o_keys), k.data(), 12ull * n, cudaMemcpyHostToDevice, 0));
	rc = b200z_pkzip_device(d.at(o_in), d.at(o_out), d.at(o_off), d.at(o_len), n, d.at(o_keys), encrypt, nullptr);
	if (rc) return rc;
	for (int i = 0; i < n; i++)
		if (len[i]) B200Z_CUDA(cudaMemcpyAsync(out[i], d.at(o_out) + off[i], (size_t)len[i], cudaMemcpyDeviceToHost, 0));
	B200Z_CUDA(cudaMemcpyAsync(k.data(), d.at(o_keys), 12ull * n, cudaMemcpyDeviceToHost, 0));
	B200Z_CUDA(cudaStreamSynchronize(0));
	for (int i = 0; i < 3 * n; i++)
		for (int b = 0; b < 4; b++) keys12[4 * i + b] = (uint8_t)(k[i] >> (8 * b));
	return B200Z_OK;
}

} // extern "C"
