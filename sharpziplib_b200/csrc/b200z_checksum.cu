// b200z_checksum.cu -- CRC-32, Adler-32 and CRC-32/BZIP2 as tile-parallel reductions (replaces Crc32.Update,
// Checksum/Crc32.cs:138-159 + CrcUtilities.cs:94-156, Adler32.Update, Checksum/Adler32.cs:134-161, and BZip2Crc.Update,
// Checksum/BZip2Crc.cs:99-169 + CrcUtilities.cs:69-77).  Kind 0 = CRC-32, 1 = Adler-32, 2 = CRC-32/BZIP2.
// One CTA per 32 KiB tile, one 128-byte chunk per thread; the combination identities are in b200z_crc.cuh.
#include "b200z_crc.cuh"
#include <mutex>

#include "b200z_internal.cuh"

namespace b200z {

__constant__ uint32_t c_crc_tab[4][256];   // slicing-by-4 tables (the first 4 slices of the reference's 16)
__constant__ uint32_t c_xpow_chunk[kCkThreads]; // x^(8 * 128 * k)
__constant__ uint32_t c_xpow_byte[kCkChunk];    // x^(8 * r)
__constant__ uint32_t c_crcn_tab[4][256];      // CRC-32/BZIP2: slicing-by-4, normal bit order
__constant__ uint32_t c_xpown_chunk[kCkThreads]; // x^(8 * 128 * k), normal bit order
__constant__ uint32_t c_xpown_byte[kCkChunk];    // x^(8 * r), normal bit order
static unsigned long long g_tables_ready = 0; // bit d: the constant tables of device d are loaded

int checksum_init_tables() {
	int dev = 0;
	B200Z_CUDA(cudaGetDevice(&dev));
	static std::mutex mu;
	std::lock_guard<std::mutex> lk(mu);
	if (dev < 64 && ((g_tables_ready >> dev) & 1ull)) return B200Z_OK;
	static uint32_t tab[4][256];
	for (uint32_t i = 0; i < 256; i++) {
		uint32_t res = i;
		for (int j = 0; j < 4; j++) {
			for (int k = 0; k < 8; k++) res = (res & 1) ? kCrcPoly ^ (res >> 1) : res >> 1;
			tab[j][i] = res;
		}
	}
	static uint32_t xc[kCkThreads], xb[kCkChunk];
	for (int k = 0; k < kCkThreads; k++) xc[k] = crc_xpow8((uint64_t)kCkChunk * k);
	for (int r = 0; r < kCkChunk; r++) xb[r] = crc_xpow8((uint64_t)r);
	B200Z_CUDA(cudaMemcpyToSymbol(c_crc_tab, tab, sizeof(tab)));
	B200Z_CUDA(cudaMemcpyToSymbol(c_xpow_chunk, xc, sizeof(xc)));
	B200Z_CUDA(cudaMemcpyToSymbol(c_xpow_byte, xb, sizeof(xb)));
	// CRC-32/BZIP2: slice j advances a byte through 8 (j + 1) shifts, as GenerateSlicingLookupTable(isReversed: false) does
	for (uint32_t i = 0; i < 256; i++) tab[0][i] = crcn_table0_entry(i);
	for (int j = 1; j < 4; j++)
		for (uint32_t i = 0; i < 256; i++) tab[j][i] = (tab[j - 1][i] << 8) ^ tab[0][tab[j - 1][i] >> 24];
	for (int k = 0; k < kCkThreads; k++) xc[k] = crcn_xpow8((uint64_t)kCkChunk * k);
	for (int r = 0; r < kCkChunk; r++) xb[r] = crcn_xpow8((uint64_t)r);
	B200Z_CUDA(cudaMemcpyToSymbol(c_crcn_tab, tab, sizeof(tab)));
	B200Z_CUDA(cudaMemcpyToSymbol(c_xpown_chunk, xc, sizeof(xc)));
	B200Z_CUDA(cudaMemcpyToSymbol(c_xpown_byte, xb, sizeof(xb)));
	if (dev < 64) g_tables_ready |= 1ull << dev;
	return B200Z_OK;
}

// tile list for n streams, with each tile's multiplier for `kind`.  Kind 2 has no dynamic (inflate) caller: refused.
int checksum_tiles(const int64_t *len, int32_t n, std::vector<CkTile> &tiles, int kind, bool dynamic) {
	tiles.clear();
	if (kind == 2 && dynamic) {
		set_error("checksum kind 2 has no tiles over capacities");
		return B200Z_E_INTERNAL;
	}
	for (int32_t i = 0; i < n; i++) {
		const int64_t L = len[i];
		const size_t first = tiles.size();
		for (int64_t s = 0; s < L; s += kCkTile) tiles.push_back(CkTile{(uint64_t)s, i, 0u});
		if (dynamic) continue; // len[] are capacities: the kernel works the multipliers out from the device-side lengths
		// multipliers from the last tile backwards: one mulmod per tile
		uint32_t m = kind == 2 ? 1u : 1u << 31; // x^0
		uint64_t after = 0;
		const uint32_t xtile = kind == 2 ? crcn_xpow8(kCkTile) : crc_xpow8(kCkTile);
		for (size_t t = tiles.size(); t-- > first;) {
			const uint64_t tlen = (uint64_t)L - tiles[t].start < (uint64_t)kCkTile ? (uint64_t)L - tiles[t].start : (uint64_t)kCkTile;
			tiles[t].mult = kind != 1 ? m : (uint32_t)(after % kAdlerBase);
			after += tlen;
			if (kind == 0) m = crc_mulmod(tlen == (uint64_t)kCkTile ? xtile : crc_xpow8(tlen), m);
			if (kind == 2) m = crcn_mulmod(tlen == (uint64_t)kCkTile ? xtile : crcn_xpow8(tlen), m);
		}
	}
	return B200Z_OK;
}

// the GF(2) arithmetic of a CRC kind: 0 reflected (CRC-32), 2 normal (CRC-32/BZIP2)
template <int KIND>
__device__ __forceinline__ uint32_t ck_mulmod(uint32_t a, uint32_t b) {
	return KIND == 0 ? crc_mulmod(a, b) : crcn_mulmod(a, b);
}
template <int KIND>
__device__ __forceinline__ uint32_t ck_xpow8(uint64_t nbytes) {
	return KIND == 0 ? crc_xpow8(nbytes) : crcn_xpow8(nbytes);
}

__global__ void k_ck_zero(uint64_t *acc, int n2) {
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n2) acc[i] = 0;
}

template <int KIND>
__global__ void __launch_bounds__(kCkThreads)
    k_checksum(const uint8_t *__restrict__ data, const int64_t *__restrict__ off, const int64_t *__restrict__ len,
               const CkTile *__restrict__ tiles, int dynamic, unsigned long long *__restrict__ acc) {
	__shared__ uint32_t s_words[kCkThreads * 33];
	__shared__ uint32_t s_tab[4][256];
	__shared__ unsigned long long s_red[2][kCkThreads / 32];
	CkTile td = tiles[blockIdx.x];
	const uint64_t n = (uint64_t)len[td.stream];
	if (td.start >= n) return; // tiles laid out for a capacity (inflate output): nothing of this stream here
	const uint8_t *src = data + off[td.stream] + td.start;
	const uint32_t tlen = n - td.start < (uint64_t)kCkTile ? (uint32_t)(n - td.start) : (uint32_t)kCkTile;
	if (KIND != 2 && dynamic) {
		// the length was not known when the tiles were made: derive the multiplier from the bytes behind this tile
		const uint64_t after = n - (td.start + tlen);
		td.mult = KIND == 0 ? crc_xpow8(after) : (uint32_t)(after % kAdlerBase);
	}
	const int tid = threadIdx.x;
	if (KIND != 1) {
		const uint32_t *tab = KIND == 0 ? &c_crc_tab[0][0] : &c_crcn_tab[0][0];
		for (int i = tid; i < 1024; i += kCkThreads) (&s_tab[0][0])[i] = tab[i];
	}
	// coalesced staging; chunk c occupies words [33c, 33c + 32)  (the +1 skew keeps the per-thread walk conflict free)
	const uint32_t nwords = (tlen + 3) >> 2;
	const uint32_t nvec = ((reinterpret_cast<uintptr_t>(src) & 15) == 0) ? (tlen >> 4) : 0u; // caller blobs may be unaligned
	const uint4 *vsrc = reinterpret_cast<const uint4 *>(src);
	for (uint32_t v = tid; v < nvec; v += kCkThreads) {
		const uint4 q = __ldg(vsrc + v);
		const uint32_t w = v << 2;
		uint32_t *d = &s_words[(w >> 5) * 33 + (w & 31)];
		d[0] = q.x;
		d[1] = q.y;
		d[2] = q.z;
		d[3] = q.w;
	}
	for (uint32_t w = (nvec << 2) + tid; w < nwords; w += kCkThreads) {
		uint32_t v = 0;
		for (uint32_t k = 0; k < 4; k++) {
			const uint32_t bi = (w << 2) + k;
			if (bi < tlen) v |= (uint32_t)src[bi] << (8 * k);
		}
		s_words[(w >> 5) * 33 + (w & 31)] = v;
	}
	__syncthreads();
	const uint32_t cstart = (uint32_t)tid * kCkChunk;
	const uint32_t clen = cstart >= tlen ? 0u : (tlen - cstart < (uint32_t)kCkChunk ? tlen - cstart : (uint32_t)kCkChunk);
	const uint32_t *cw = &s_words[tid * 33];
	const uint32_t K = tlen / kCkChunk, r = tlen % kCkChunk; // full chunks, bytes in the partial chunk
	if (KIND != 1) {
		uint32_t c = 0;
		const uint32_t fw = clen >> 2;
		if (KIND == 0) {
			for (uint32_t i = 0; i < fw; i++) {
				const uint32_t x = c ^ cw[i];
				c = s_tab[3][x & 0xFF] ^ s_tab[2][(x >> 8) & 0xFF] ^ s_tab[1][(x >> 16) & 0xFF] ^ s_tab[0][x >> 24];
			}
			if (clen & 3) {
				uint32_t w = cw[fw];
				for (uint32_t k = 0; k < (clen & 3); k++) {
					c = s_tab[0][(c ^ w) & 0xFF] ^ (c >> 8);
					w >>= 8;
				}
			}
		} else {
			// the words are little-endian: byte-swapped, the first byte of each lands in the top of the register
			for (uint32_t i = 0; i < fw; i++) {
				const uint32_t x = c ^ __byte_perm(cw[i], 0, 0x0123);
				c = s_tab[3][x >> 24] ^ s_tab[2][(x >> 16) & 0xFF] ^ s_tab[1][(x >> 8) & 0xFF] ^ s_tab[0][x & 0xFF];
			}
			if (clen & 3) {
				uint32_t w = cw[fw];
				for (uint32_t k = 0; k < (clen & 3); k++) {
					c = s_tab[0][((c >> 24) ^ w) & 0xFF] ^ (c << 8);
					w >>= 8;
				}
			}
		}
		// shift to the end of the tile: full chunks by x^(8*128*(K-1-t)) then x^(8r); the partial chunk not at all
		const uint32_t *xpow_chunk = KIND == 0 ? c_xpow_chunk : c_xpown_chunk;
		const uint32_t *xpow_byte = KIND == 0 ? c_xpow_byte : c_xpown_byte;
		uint32_t contrib = 0;
		if (clen == (uint32_t)kCkChunk) contrib = ck_mulmod<KIND>(xpow_chunk[K - 1 - tid], c);
		for (int o = 16; o > 0; o >>= 1) contrib ^= __shfl_xor_sync(0xffffffffu, contrib, o);
		if ((tid & 31) == 0) s_red[0][tid >> 5] = contrib;
		if (clen > 0 && clen < (uint32_t)kCkChunk) s_red[1][0] = c; // exactly one thread owns the partial chunk
		__syncthreads();
		if (tid == 0) {
			uint32_t R = 0;
			for (int k = 0; k < kCkThreads / 32; k++) R ^= (uint32_t)s_red[0][k];
			if (r) R = ck_mulmod<KIND>(xpow_byte[r], R) ^ (uint32_t)s_red[1][0];
			R = ck_mulmod<KIND>(td.mult, R);
			atomicXor(reinterpret_cast<unsigned int *>(&acc[2 * td.stream]), R);
		}
	} else {
		uint32_t A = 0, B = 0;
		const uint32_t fw = (clen + 3) >> 2;
		uint32_t left = clen;
		for (uint32_t i = 0; i < fw; i++) {
			uint32_t w = cw[i];
			for (int k = 0; k < 4 && left > 0; k++, left--) {
				const uint32_t b = w & 0xFF;
				w >>= 8;
				A += b;
				B += left * b; // weight = bytes from this one to the end of the chunk
			}
		}
		// bytes after this chunk inside the tile
		const uint32_t after = tlen - (cstart + clen);
		unsigned long long a64 = A, b64 = (unsigned long long)B + (unsigned long long)A * (clen ? after : 0u);
		for (int o = 16; o > 0; o >>= 1) {
			a64 += __shfl_xor_sync(0xffffffffu, a64, o);
			b64 += __shfl_xor_sync(0xffffffffu, b64, o);
		}
		if ((tid & 31) == 0) {
			s_red[0][tid >> 5] = a64;
			s_red[1][tid >> 5] = b64;
		}
		__syncthreads();
		if (tid == 0) {
			unsigned long long As = 0, Bs = 0;
			for (int k = 0; k < kCkThreads / 32; k++) {
				As += s_red[0][k];
				Bs += s_red[1][k];
			}
			As %= kAdlerBase;
			Bs = (Bs + As * (unsigned long long)td.mult) % kAdlerBase;
			atomicAdd(&acc[2 * td.stream], As);
			atomicAdd(&acc[2 * td.stream + 1], Bs);
		}
	}
	(void)K;
}

template <int KIND>
__global__ void k_ck_final(const int64_t *__restrict__ len, int n, const unsigned long long *__restrict__ acc,
                           uint32_t *__restrict__ value, int fresh) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint64_t L = (uint64_t)len[i];
	if (KIND != 1) {
		const uint32_t v0 = fresh ? 0u : value[i];
		const uint32_t reg = v0 ^ 0xFFFFFFFFu;
		value[i] = (ck_mulmod<KIND>(ck_xpow8<KIND>(L), reg) ^ (uint32_t)acc[2 * i]) ^ 0xFFFFFFFFu;
	} else {
		const uint32_t v0 = fresh ? 1u : value[i];
		const unsigned long long s1 = v0 & 0xFFFFu, s2 = v0 >> 16;
		const unsigned long long n1 = (s1 + acc[2 * i]) % kAdlerBase;
		const unsigned long long n2 = (s2 + (L % kAdlerBase) * s1 + acc[2 * i + 1]) % kAdlerBase;
		value[i] = (uint32_t)((n2 << 16) | n1);
	}
}

// acc: 2 x uint64 per stream of scratch
int checksum_launch(int kind, const uint8_t *d_data, const int64_t *d_off, const int64_t *d_len, int32_t n,
                    const CkTile *d_tiles, int32_t n_tiles, unsigned long long *d_acc, uint32_t *d_value, int fresh,
                    cudaStream_t s, bool dynamic) {
	if (kind == 2 && dynamic) {
		set_error("checksum kind 2 has no tiles over capacities");
		return B200Z_E_INTERNAL;
	}
	int rc = checksum_init_tables();
	if (rc) return rc;
	if (n == 0) return B200Z_OK;
	k_ck_zero<<<(2 * n + 255) / 256, 256, 0, s>>>(reinterpret_cast<uint64_t *>(d_acc), 2 * n);
	if (n_tiles) {
		if (kind == 0) k_checksum<0><<<n_tiles, kCkThreads, 0, s>>>(d_data, d_off, d_len, d_tiles, dynamic ? 1 : 0, d_acc);
		else if (kind == 1) k_checksum<1><<<n_tiles, kCkThreads, 0, s>>>(d_data, d_off, d_len, d_tiles, dynamic ? 1 : 0, d_acc);
		else k_checksum<2><<<n_tiles, kCkThreads, 0, s>>>(d_data, d_off, d_len, d_tiles, 0, d_acc);
	}
	if (kind == 0) k_ck_final<0><<<(n + 127) / 128, 128, 0, s>>>(d_len, n, d_acc, d_value, fresh);
	else if (kind == 1) k_ck_final<1><<<(n + 127) / 128, 128, 0, s>>>(d_len, n, d_acc, d_value, fresh);
	else k_ck_final<2><<<(n + 127) / 128, 128, 0, s>>>(d_len, n, d_acc, d_value, fresh);
	B200Z_CUDA(cudaGetLastError());
	return B200Z_OK;
}

} // namespace b200z
