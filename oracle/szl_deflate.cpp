// szl_deflate.cpp -- ORACLE (test infrastructure): checksums + Deflater side.
// Restates Checksum/{Adler32,Crc32,CrcUtilities}.cs and
// Zip/Compression/{PendingBuffer,DeflaterPending,DeflaterConstants,DeflaterHuffman,
// DeflaterEngine,Deflater}.cs of the reference (paths relative to
// SharpZipLib's src/ICSharpCode.SharpZipLib/).  See szl_oracle.hpp for the pinning status.
#include "szl_oracle.hpp"
#include <algorithm>
#include <cstring>

namespace szl {

// ============================== Checksum/Adler32.cs =======================================
static const uint32_t ADLER_BASE = 65521; // Adler32.cs:56

void Adler32::Update(int bval) { // Adler32.cs:96-108
	uint32_t s1 = checkValue & 0xFFFF;
	uint32_t s2 = checkValue >> 16;
	s1 = (s1 + ((uint32_t)bval & 0xFF)) % ADLER_BASE;
	s2 = (s1 + s2) % ADLER_BASE;
	checkValue = (s2 << 16) + s1;
}

void Adler32::Update(const uint8_t *buf, size_t offset, size_t count) { // Adler32.cs:134-161
	uint32_t s1 = checkValue & 0xFFFF;
	uint32_t s2 = checkValue >> 16;
	while (count > 0) {
		// deferred modulo: at most 3800 bytes between reductions
		size_t n = 3800;
		if (n > count) n = count;
		count -= n;
		while (n-- > 0) {
			s1 = s1 + (uint32_t)(buf[offset++] & 0xff);
			s2 = s2 + s1;
		}
		s1 %= ADLER_BASE;
		s2 %= ADLER_BASE;
	}
	checkValue = (s2 << 16) | s1;
}

// ============================== Checksum/CrcUtilities.cs + Crc32.cs =======================
static const int SlicingDegree = 16; // CrcUtilities.cs:10

static const uint32_t *crcTable() { // CrcUtilities.cs:25-52 (isReversed == true branch), Crc32.cs:50
	static uint32_t table[256 * SlicingDegree];
	static bool init = false;
	if (!init) {
		const uint32_t polynomial = 0xEDB88320u;
		const uint32_t one = 1;
		for (int i = 0; i < 256; i++) {
			uint32_t res = (uint32_t)i;
			for (int j = 0; j < SlicingDegree; j++) {
				for (int k = 0; k < 8; k++) {
					res = (res & one) == 1 ? polynomial ^ (res >> 1) : res >> 1;
				}
				table[(256 * j) + i] = res;
			}
		}
		init = true;
	}
	return table;
}

void Crc32::Update(int bval) { // Crc32.cs:100-103
	const uint32_t *t = crcTable();
	checkValue = t[(checkValue ^ (uint32_t)bval) & 0xFF] ^ (checkValue >> 8);
}

// CrcUtilities.cs:94-101 + :134-156
static inline uint32_t UpdateDataForReversedPoly(const uint8_t *input, size_t offset, const uint32_t *t, uint32_t checkValue) {
	uint8_t x1 = (uint8_t)((uint8_t)checkValue ^ input[offset]);
	uint8_t x2 = (uint8_t)((uint8_t)(checkValue >>= 8) ^ input[offset + 1]);
	uint8_t x3 = (uint8_t)((uint8_t)(checkValue >>= 8) ^ input[offset + 2]);
	uint8_t x4 = (uint8_t)((uint8_t)(checkValue >>= 8) ^ input[offset + 3]);
	uint32_t result;
	uint32_t a1 = t[x1 + 3840] ^ t[x2 + 3584];
	uint32_t a2 = t[x3 + 3328] ^ t[x4 + 3072];
	result = t[input[offset + 4] + 2816];
	result ^= t[input[offset + 5] + 2560];
	a1 ^= t[input[offset + 9] + 1536];
	result ^= t[input[offset + 6] + 2304];
	result ^= t[input[offset + 7] + 2048];
	result ^= t[input[offset + 8] + 1792];
	a2 ^= t[input[offset + 13] + 512];
	result ^= t[input[offset + 10] + 1280];
	result ^= t[input[offset + 11] + 1024];
	result ^= t[input[offset + 12] + 768];
	result ^= a1;
	result ^= t[input[offset + 14] + 256];
	result ^= t[input[offset + 15]];
	result ^= a2;
	return result;
}

void Crc32::Update(const uint8_t *data, size_t offset, size_t count) { // Crc32.cs:138-159
	const uint32_t *t = crcTable();
	size_t remainder = count % SlicingDegree;
	size_t end = offset + count - remainder;
	while (offset != end) {
		checkValue = UpdateDataForReversedPoly(data, offset, t, checkValue);
		offset += SlicingDegree;
	}
	if (remainder != 0) {
		size_t e2 = end + remainder; // SlowUpdateLoop, Crc32.cs:165-171
		while (offset != e2) Update(data[offset++]);
	}
}

// ============================== Zip/Compression/PendingBuffer.cs ==========================
void PendingBuffer::WriteBlock(const uint8_t *block, int offset, int length) { // :115-127
	if (end + length > (int)buffer.size()) throw SzlError(E_INTERNAL, "PendingBuffer overflow (WriteBlock)");
	std::memcpy(&buffer[end], block + offset, (size_t)length);
	end += length;
}

void PendingBuffer::AlignToByte() { // :143-161
	if (bitCount > 0) {
		put((uint8_t)bits);
		if (bitCount > 8) put((uint8_t)(bits >> 8));
	}
	bits = 0;
	bitCount = 0;
}

void PendingBuffer::WriteBits(int b, int count) { // :168-189
	bits |= (uint32_t)(b << bitCount);
	bitCount += count;
	if (bitCount >= 16) {
		put((uint8_t)bits);
		put((uint8_t)(bits >> 8));
		bits >>= 16;
		bitCount -= 16;
	}
}

int PendingBuffer::Flush(uint8_t *output, int offset, int length) { // :226-248
	if (bitCount >= 8) {
		put((uint8_t)bits);
		bits >>= 8;
		bitCount -= 8;
	}
	if (length > end - start) {
		length = end - start;
		std::memcpy(output + offset, &buffer[start], (size_t)length);
		start = 0;
		end = 0;
	} else {
		std::memcpy(output + offset, &buffer[start], (size_t)length);
		start += length;
	}
	return length;
}

// ============================== Zip/Compression/DeflaterConstants.cs ======================
namespace DC {
static const int STORED_BLOCK = 0, STATIC_TREES = 1, DYN_TREES = 2, PRESET_DICT = 0x20;
static const int DEFAULT_MEM_LEVEL = 8;
static const int MAX_MATCH = 258, MIN_MATCH = 3, MAX_WBITS = 15;
static const int WSIZE = 1 << MAX_WBITS, WMASK = WSIZE - 1;
static const int HASH_BITS = DEFAULT_MEM_LEVEL + 7, HASH_SIZE = 1 << HASH_BITS, HASH_MASK = HASH_SIZE - 1;
static const int HASH_SHIFT = (HASH_BITS + MIN_MATCH - 1) / MIN_MATCH;
static const int MIN_LOOKAHEAD = MAX_MATCH + MIN_MATCH + 1;
static const int MAX_DIST = WSIZE - MIN_LOOKAHEAD;
static const int PENDING_BUF_SIZE = 1 << (DEFAULT_MEM_LEVEL + 8);
static const int MAX_BLOCK_SIZE = (65535 < PENDING_BUF_SIZE - 5) ? 65535 : PENDING_BUF_SIZE - 5;
static const int DEFLATE_STORED = 0, DEFLATE_FAST = 1, DEFLATE_SLOW = 2;
static const int GOOD_LENGTH[] = {0, 4, 4, 4, 4, 8, 8, 8, 32, 32};          // :124
static const int MAX_LAZY[] = {0, 4, 5, 6, 4, 16, 16, 32, 128, 258};        // :129
static const int NICE_LENGTH[] = {0, 8, 16, 32, 16, 32, 128, 128, 258, 258}; // :134
static const int MAX_CHAIN[] = {0, 4, 8, 32, 16, 32, 128, 256, 1024, 4096};  // :139
static const int COMPR_FUNC[] = {0, 1, 1, 1, 1, 2, 2, 2, 2, 2};              // :144
} // namespace DC

// ============================== Zip/Compression/DeflaterHuffman.cs ========================
static const int REP_3_6 = 16, REP_3_10 = 17, REP_11_138 = 18, EOF_SYMBOL = 256;
static const int BL_ORDER[] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15}; // :34
static const uint8_t bit4Reverse[] = {0, 8, 4, 12, 2, 10, 6, 14, 1, 9, 5, 13, 3, 11, 7, 15};        // :36-53

int16_t DeflaterHuffman::BitReverse(int toReverse) { // :924-930
	return (int16_t)(bit4Reverse[toReverse & 0xF] << 12 | bit4Reverse[(toReverse >> 4) & 0xF] << 8 |
	                 bit4Reverse[(toReverse >> 8) & 0xF] << 4 | bit4Reverse[toReverse >> 12]);
}

struct StaticCodes { // static ctor, :602-642
	int16_t staticLCodes[DeflaterHuffman::LITERAL_NUM];
	uint8_t staticLLength[DeflaterHuffman::LITERAL_NUM];
	int16_t staticDCodes[DeflaterHuffman::DIST_NUM];
	uint8_t staticDLength[DeflaterHuffman::DIST_NUM];
	StaticCodes() {
		int i = 0;
		while (i < 144) { staticLCodes[i] = DeflaterHuffman::BitReverse((0x030 + i) << 8); staticLLength[i++] = 8; }
		while (i < 256) { staticLCodes[i] = DeflaterHuffman::BitReverse((0x190 - 144 + i) << 7); staticLLength[i++] = 9; }
		while (i < 280) { staticLCodes[i] = DeflaterHuffman::BitReverse((0x000 - 256 + i) << 9); staticLLength[i++] = 7; }
		while (i < DeflaterHuffman::LITERAL_NUM) { staticLCodes[i] = DeflaterHuffman::BitReverse((0x0c0 - 280 + i) << 8); staticLLength[i++] = 8; }
		for (i = 0; i < DeflaterHuffman::DIST_NUM; i++) { staticDCodes[i] = DeflaterHuffman::BitReverse(i << 11); staticDLength[i] = 5; }
	}
};
static const StaticCodes &statics() { static StaticCodes s; return s; }

DeflaterHuffman::Tree::Tree(DeflaterHuffman *dh_, int elems, int minCodes, int maxLength_) // :85-92
	: freqs(elems, 0), minNumCodes(minCodes), bl_counts(maxLength_, 0), maxLength(maxLength_), dh(dh_) {}

void DeflaterHuffman::Tree::Reset() { // :99-107
	for (size_t i = 0; i < freqs.size(); i++) freqs[i] = 0;
	codes.clear();
	length.clear();
	haveLength = false;
}

void DeflaterHuffman::Tree::WriteSymbol(int code) { // :109-116
	dh->pending->WriteBits(codes[code] & 0xffff, length[code]);
}

void DeflaterHuffman::Tree::SetStaticCodes(const int16_t *staticCodes, const uint8_t *staticLengths, int n) { // :142-146
	codes.assign(staticCodes, staticCodes + n);
	length.assign(staticLengths, staticLengths + n);
	haveLength = true;
}

void DeflaterHuffman::Tree::BuildCodes() { // :151-194
	std::vector<int> nextCode(maxLength);
	int code = 0;
	codes.assign(freqs.size(), 0);
	for (int bits = 0; bits < maxLength; bits++) {
		nextCode[bits] = code;
		code += bl_counts[bits] << (15 - bits);
	}
	for (int i = 0; i < numCodes; i++) {
		int bits = length[i];
		if (bits > 0) {
			codes[i] = BitReverse(nextCode[bits - 1]);
			nextCode[bits - 1] += 1 << (16 - bits);
		}
	}
}

void DeflaterHuffman::Tree::BuildTree() { // :196-329
	int numSymbols = (int)freqs.size();
	// heap: priority queue on frequency; 0 is the root, 2n+1 / 2n+2 the children of n
	std::vector<int> heap(numSymbols);
	int heapLen = 0;
	int maxCode = 0;
	for (int n = 0; n < numSymbols; n++) {
		int freq = freqs[n];
		if (freq != 0) {
			// insert n into heap
			int pos = heapLen++;
			int ppos;
			while (pos > 0 && freqs[heap[ppos = (pos - 1) / 2]] > freq) {
				heap[pos] = heap[ppos];
				pos = ppos;
			}
			heap[pos] = n;
			maxCode = n;
		}
	}
	// force at least two codes (:235-239)
	while (heapLen < 2) {
		int node = maxCode < 2 ? ++maxCode : 0;
		heap[heapLen++] = node;
	}
	numCodes = std::max(maxCode + 1, minNumCodes);
	int numLeafs = heapLen;
	std::vector<int> childs(4 * heapLen - 2);
	std::vector<int> values(2 * heapLen - 1);
	int numNodes = numLeafs;
	for (int i = 0; i < heapLen; i++) {
		int node = heap[i];
		childs[2 * i] = node;
		childs[2 * i + 1] = -1;
		values[i] = freqs[node] << 8;
		heap[i] = i;
	}
	// combine the two least frequent nodes until one is left (:259-321)
	do {
		int first = heap[0];
		int last = heap[--heapLen];
		// propagate the hole to the leafs of the heap
		int ppos = 0;
		int path = 1;
		while (path < heapLen) {
			if (path + 1 < heapLen && values[heap[path]] > values[heap[path + 1]]) path++;
			heap[ppos] = heap[path];
			ppos = path;
			path = path * 2 + 1;
		}
		// now propagate the last element down along path
		int lastVal = values[last];
		while ((path = ppos) > 0 && values[heap[ppos = (path - 1) / 2]] > lastVal) heap[path] = heap[ppos];
		heap[path] = last;

		int second = heap[0];
		// create a new node father of first and second
		last = numNodes++;
		childs[2 * last] = first;
		childs[2 * last + 1] = second;
		int mindepth = std::min(values[first] & 0xff, values[second] & 0xff);
		values[last] = lastVal = values[first] + values[second] - mindepth + 1;
		// again, propagate the hole to the leafs
		ppos = 0;
		path = 1;
		while (path < heapLen) {
			if (path + 1 < heapLen && values[heap[path]] > values[heap[path + 1]]) path++;
			heap[ppos] = heap[path];
			ppos = path;
			path = ppos * 2 + 1;
		}
		// now propagate the new element down along path
		while ((path = ppos) > 0 && values[heap[ppos = (path - 1) / 2]] > lastVal) heap[path] = heap[ppos];
		heap[path] = last;
	} while (heapLen > 1);
	if (heap[0] != (int)childs.size() / 2 - 1) throw SzlError(E_DATA, "Heap invariant violated");
	BuildLength(childs);
}

int DeflaterHuffman::Tree::GetEncodedLength() const { // :335-343
	int len = 0;
	for (size_t i = 0; i < freqs.size(); i++) len += freqs[i] * length[i];
	return len;
}

void DeflaterHuffman::Tree::CalcBLFreq(Tree &blTree) { // :349-405
	int max_count, min_count, count;
	int curlen = -1;
	int i = 0;
	while (i < numCodes) {
		count = 1;
		int nextlen = length[i];
		if (nextlen == 0) {
			max_count = 138;
			min_count = 3;
		} else {
			max_count = 6;
			min_count = 3;
			if (curlen != nextlen) {
				blTree.freqs[nextlen]++;
				count = 0;
			}
		}
		curlen = nextlen;
		i++;
		while (i < numCodes && curlen == length[i]) {
			i++;
			if (++count >= max_count) break;
		}
		if (count < min_count) blTree.freqs[curlen] += (int16_t)count;
		else if (curlen != 0) blTree.freqs[REP_3_6]++;
		else if (count <= 10) blTree.freqs[REP_3_10]++;
		else blTree.freqs[REP_11_138]++;
	}
}

void DeflaterHuffman::Tree::WriteTree(Tree &blTree) { // :411-473
	int max_count, min_count, count;
	int curlen = -1;
	int i = 0;
	while (i < numCodes) {
		count = 1;
		int nextlen = length[i];
		if (nextlen == 0) {
			max_count = 138;
			min_count = 3;
		} else {
			max_count = 6;
			min_count = 3;
			if (curlen != nextlen) {
				blTree.WriteSymbol(nextlen);
				count = 0;
			}
		}
		curlen = nextlen;
		i++;
		while (i < numCodes && curlen == length[i]) {
			i++;
			if (++count >= max_count) break;
		}
		if (count < min_count) {
			while (count-- > 0) blTree.WriteSymbol(curlen);
		} else if (curlen != 0) {
			blTree.WriteSymbol(REP_3_6);
			dh->pending->WriteBits(count - 3, 2);
		} else if (count <= 10) {
			blTree.WriteSymbol(REP_3_10);
			dh->pending->WriteBits(count - 3, 3);
		} else {
			blTree.WriteSymbol(REP_11_138);
			dh->pending->WriteBits(count - 11, 7);
		}
	}
}

void DeflaterHuffman::Tree::BuildLength(const std::vector<int> &childs) { // :475-579
	length.assign(freqs.size(), 0);
	haveLength = true;
	int numNodes = (int)childs.size() / 2;
	int numLeafs = (numNodes + 1) / 2;
	int overflow = 0;
	for (int i = 0; i < maxLength; i++) bl_counts[i] = 0;
	// first calculate optimal bit lengths
	std::vector<int> lengths(numNodes);
	lengths[numNodes - 1] = 0;
	for (int i = numNodes - 1; i >= 0; i--) {
		if (childs[2 * i + 1] != -1) {
			int bitLength = lengths[i] + 1;
			if (bitLength > maxLength) {
				bitLength = maxLength;
				overflow++;
			}
			lengths[childs[2 * i]] = lengths[childs[2 * i + 1]] = bitLength;
		} else {
			// a leaf node
			int bitLength = lengths[i];
			bl_counts[bitLength - 1]++;
			length[childs[2 * i]] = (uint8_t)lengths[i];
		}
	}
	if (overflow == 0) return;
	int incrBitLen = maxLength - 1;
	do {
		// find the first bit length which could increase
		while (bl_counts[--incrBitLen] == 0) {
		}
		// move this node one down and remove a corresponding number of overflow nodes
		do {
			bl_counts[incrBitLen]--;
			bl_counts[++incrBitLen]++;
			overflow -= 1 << (maxLength - 1 - incrBitLen);
		} while (overflow > 0 && incrBitLen < maxLength - 1);
	} while (overflow > 0);
	// we may have overshot above
	bl_counts[maxLength - 1] += overflow;
	bl_counts[maxLength - 2] -= overflow;
	// recompute all bit lengths, scanning in increasing frequency (:557-571)
	int nodePtr = 2 * numLeafs;
	for (int bits = maxLength; bits != 0; bits--) {
		int n = bl_counts[bits - 1];
		while (n > 0) {
			int childPtr = 2 * childs[nodePtr++];
			if (childs[childPtr + 1] == -1) {
				// we found another leaf
				length[childs[childPtr]] = (uint8_t)bits;
				n--;
			}
		}
	}
}

DeflaterHuffman::DeflaterHuffman(PendingBuffer *pending_) // :648-658
	: pending(pending_), literalTree(this, LITERAL_NUM, 257, 15), distTree(this, DIST_NUM, 1, 15),
	  blTree(this, BITLEN_NUM, 4, 7), d_buf(BUFSIZE), l_buf(BUFSIZE) {}

void DeflaterHuffman::Reset() { // :663-670
	last_lit = 0;
	extra_bits = 0;
	literalTree.Reset();
	distTree.Reset();
	blTree.Reset();
}

void DeflaterHuffman::SendAllTrees(int blTreeCodes) { // :676-696
	blTree.BuildCodes();
	literalTree.BuildCodes();
	distTree.BuildCodes();
	pending->WriteBits(literalTree.numCodes - 257, 5);
	pending->WriteBits(distTree.numCodes - 1, 5);
	pending->WriteBits(blTreeCodes - 4, 4);
	for (int rank = 0; rank < blTreeCodes; rank++) pending->WriteBits(blTree.length[BL_ORDER[rank]], 3);
	literalTree.WriteTree(blTree);
	distTree.WriteTree(blTree);
}

void DeflaterHuffman::CompressBlock() { // :701-757
	for (int i = 0; i < last_lit; i++) {
		int litlen = l_buf[i] & 0xff;
		int dist = d_buf[i];
		if (dist-- != 0) {
			int lc = Lcode(litlen);
			literalTree.WriteSymbol(lc);
			int bits = (lc - 261) / 4;
			if (bits > 0 && bits <= 5) pending->WriteBits(litlen & ((1 << bits) - 1), bits);
			int dc = Dcode(dist);
			distTree.WriteSymbol(dc);
			bits = dc / 2 - 1;
			if (bits > 0) pending->WriteBits(dist & ((1 << bits) - 1), bits);
		} else {
			literalTree.WriteSymbol(litlen);
		}
	}
	literalTree.WriteSymbol(EOF_SYMBOL);
}

void DeflaterHuffman::FlushStoredBlock(const uint8_t *stored, int storedOffset, int storedLength, bool lastBlock) { // :766-779
	if (trace) trace->push_back({0, last_lit, storedLength, -1, -1});
	pending->WriteBits((DC::STORED_BLOCK << 1) + (lastBlock ? 1 : 0), 3);
	pending->AlignToByte();
	pending->WriteShort(storedLength);
	pending->WriteShort(~storedLength);
	pending->WriteBlock(stored, storedOffset, storedLength);
	Reset();
}

void DeflaterHuffman::FlushBlock(const uint8_t *stored, int storedOffset, int storedLength, bool lastBlock) { // :788-857
	literalTree.freqs[EOF_SYMBOL]++;
	// build trees
	literalTree.BuildTree();
	distTree.BuildTree();
	// calculate bitlen frequency
	literalTree.CalcBLFreq(blTree);
	distTree.CalcBLFreq(blTree);
	// build bitlen tree
	blTree.BuildTree();
	int blTreeCodes = 4;
	for (int i = 18; i > blTreeCodes; i--) {
		if (blTree.length[BL_ORDER[i]] > 0) blTreeCodes = i + 1;
	}
	int opt_len = 14 + blTreeCodes * 3 + blTree.GetEncodedLength() + literalTree.GetEncodedLength() +
	              distTree.GetEncodedLength() + extra_bits;
	int static_len = extra_bits;
	const StaticCodes &st = statics();
	for (int i = 0; i < LITERAL_NUM; i++) static_len += literalTree.freqs[i] * st.staticLLength[i];
	for (int i = 0; i < DIST_NUM; i++) static_len += distTree.freqs[i] * st.staticDLength[i];
	if (opt_len >= static_len) opt_len = static_len; // force static trees
	if (storedOffset >= 0 && storedLength + 4 < opt_len >> 3) {
		FlushStoredBlock(stored, storedOffset, storedLength, lastBlock);
	} else if (opt_len == static_len) {
		if (trace) trace->push_back({1, last_lit, storedLength, opt_len, static_len});
		pending->WriteBits((DC::STATIC_TREES << 1) + (lastBlock ? 1 : 0), 3);
		literalTree.SetStaticCodes(st.staticLCodes, st.staticLLength, LITERAL_NUM);
		distTree.SetStaticCodes(st.staticDCodes, st.staticDLength, DIST_NUM);
		CompressBlock();
		Reset();
	} else {
		if (trace) trace->push_back({2, last_lit, storedLength, opt_len, static_len});
		pending->WriteBits((DC::DYN_TREES << 1) + (lastBlock ? 1 : 0), 3);
		SendAllTrees(blTreeCodes);
		CompressBlock();
		Reset();
	}
}

bool DeflaterHuffman::TallyLit(int literal) { // :873-886
	d_buf[last_lit] = 0;
	l_buf[last_lit++] = (uint8_t)literal;
	literalTree.freqs[literal]++;
	return IsFull();
}

bool DeflaterHuffman::TallyDist(int distance, int length) { // :894-916
	d_buf[last_lit] = (int16_t)distance;
	l_buf[last_lit++] = (uint8_t)(length - 3);
	int lc = Lcode(length - 3);
	literalTree.freqs[lc]++;
	if (lc >= 265 && lc < 285) extra_bits += (lc - 261) / 4;
	int dc = Dcode(distance - 1);
	distTree.freqs[dc]++;
	if (dc >= 4) extra_bits += dc / 2 - 1;
	return IsFull();
}

int DeflaterHuffman::Lcode(int length) { // :932-946
	if (length == 255) return 285;
	int code = 257;
	while (length >= 8) {
		code += 4;
		length >>= 1;
	}
	return code + length;
}

int DeflaterHuffman::Dcode(int distance) { // :948-957
	int code = 0;
	while (distance >= 4) {
		code += 2;
		distance >>= 1;
	}
	return code + distance;
}

// ============================== Zip/Compression/DeflaterEngine.cs =========================
static const int TooFar = 4096; // :51

DeflaterEngine::DeflaterEngine(PendingBuffer *pending_, bool noAdlerCalculation) // :80-94
	: huffman(pending_), head(DC::HASH_SIZE, 0), prev(DC::WSIZE, 0), window(2 * DC::WSIZE, 0), pending(pending_),
	  hasAdler(!noAdlerCalculation) {
	// start at index 1: a repeat pattern cannot be built at index 0 (trap T1)
	blockStart = strstart = 1;
}

bool DeflaterEngine::Deflate(bool flush, bool finish) { // :104-137
	bool progress;
	do {
		FillWindow();
		bool canFlush = flush && (inputOff == inputEnd);
		switch (compressionFunction) {
		case DC::DEFLATE_STORED: progress = DeflateStored(canFlush, finish); break;
		case DC::DEFLATE_FAST: progress = DeflateFast(canFlush, finish); break;
		case DC::DEFLATE_SLOW: progress = DeflateSlow(canFlush, finish); break;
		default: throw SzlError(E_STATE, "unknown compressionFunction");
		}
	} while (pending->IsFlushed() && progress); // repeat while there is no pending output and progress was made
	return progress;
}

void DeflaterEngine::SetInput(const uint8_t *buffer, int offset, int count) { // :146-182
	if (buffer == nullptr) throw SzlError(E_ARG, "buffer");
	if (offset < 0) throw SzlError(E_ARG, "offset");
	if (count < 0) throw SzlError(E_ARG, "count");
	if (inputOff < inputEnd) throw SzlError(E_STATE, "Old input was not completely processed");
	int end = offset + count;
	if (offset > end) throw SzlError(E_ARG, "count");
	inputBuf = buffer;
	inputOff = offset;
	inputEnd = end;
}

void DeflaterEngine::SetDictionary(const uint8_t *buffer, int offset, int length) { // :198-229
	if (hasAdler) adler.Update(buffer, (size_t)offset, (size_t)length);
	if (length < DC::MIN_MATCH) return;
	if (length > DC::MAX_DIST) {
		offset += length - DC::MAX_DIST;
		length = DC::MAX_DIST;
	}
	std::memcpy(&window[strstart], buffer + offset, (size_t)length);
	UpdateHash();
	--length;
	while (--length > 0) {
		InsertString();
		strstart++;
	}
	strstart += 2;
	blockStart = strstart;
}

void DeflaterEngine::Reset() { // :234-253
	huffman.Reset();
	if (hasAdler) adler.Reset();
	blockStart = strstart = 1;
	lookahead = 0;
	totalIn = 0;
	prevAvailable = false;
	matchLen = DC::MIN_MATCH - 1;
	for (int i = 0; i < DC::HASH_SIZE; i++) head[i] = 0;
	for (int i = 0; i < DC::WSIZE; i++) prev[i] = 0;
}

void DeflaterEngine::SetLevel(int level) { // :304-361
	if (level < 0 || level > 9) throw SzlError(E_ARG, "level");
	goodLength = DC::GOOD_LENGTH[level];
	max_lazy = DC::MAX_LAZY[level];
	niceLength = DC::NICE_LENGTH[level];
	max_chain = DC::MAX_CHAIN[level];
	if (DC::COMPR_FUNC[level] != compressionFunction) {
		switch (compressionFunction) {
		case DC::DEFLATE_STORED:
			if (strstart > blockStart) {
				huffman.FlushStoredBlock(window.data(), blockStart, strstart - blockStart, false);
				blockStart = strstart;
			}
			UpdateHash();
			break;
		case DC::DEFLATE_FAST:
			if (strstart > blockStart) {
				huffman.FlushBlock(window.data(), blockStart, strstart - blockStart, false);
				blockStart = strstart;
			}
			break;
		case DC::DEFLATE_SLOW:
			if (prevAvailable) huffman.TallyLit(window[strstart - 1] & 0xff);
			if (strstart > blockStart) {
				huffman.FlushBlock(window.data(), blockStart, strstart - blockStart, false);
				blockStart = strstart;
			}
			prevAvailable = false;
			matchLen = DC::MIN_MATCH - 1;
			break;
		}
		compressionFunction = DC::COMPR_FUNC[level];
	}
}

void DeflaterEngine::FillWindow() { // :366-400
	// if the window is almost full and there is insufficient lookahead, slide (trap T8)
	if (strstart >= DC::WSIZE + DC::MAX_DIST) SlideWindow();
	// if there is not enough lookahead, but still some input left, read in the input
	if (lookahead < DC::MIN_LOOKAHEAD && inputOff < inputEnd) {
		int more = 2 * DC::WSIZE - lookahead - strstart;
		if (more > inputEnd - inputOff) more = inputEnd - inputOff;
		std::memcpy(&window[strstart + lookahead], inputBuf + inputOff, (size_t)more);
		if (hasAdler) adler.Update(inputBuf, (size_t)inputOff, (size_t)more);
		inputOff += more;
		totalIn += more;
		lookahead += more;
	}
	if (lookahead >= DC::MIN_MATCH) UpdateHash();
}

void DeflaterEngine::UpdateHash() { // :402-410
	ins_h = (window[strstart] << DC::HASH_SHIFT) ^ window[strstart + 1];
}

int DeflaterEngine::InsertString() { // :417-439
	int16_t match;
	int hash = ((ins_h << DC::HASH_SHIFT) ^ window[strstart + (DC::MIN_MATCH - 1)]) & DC::HASH_MASK;
	prev[strstart & DC::WMASK] = match = head[hash];
	head[hash] = (int16_t)strstart;
	ins_h = hash;
	return match & 0xffff;
}

void DeflaterEngine::SlideWindow() { // :441-462
	std::memmove(&window[0], &window[DC::WSIZE], (size_t)DC::WSIZE);
	matchStart -= DC::WSIZE;
	strstart -= DC::WSIZE;
	blockStart -= DC::WSIZE;
	// slide the hash table
	for (int i = 0; i < DC::HASH_SIZE; ++i) {
		int m = head[i] & 0xffff;
		head[i] = (int16_t)(m >= DC::WSIZE ? (m - DC::WSIZE) : 0);
	}
	// slide the prev table
	for (int i = 0; i < DC::WSIZE; i++) {
		int m = prev[i] & 0xffff;
		prev[i] = (int16_t)(m >= DC::WSIZE ? (m - DC::WSIZE) : 0);
	}
}

bool DeflaterEngine::FindLongestMatch(int curMatch) { // :474-612
	int match;
	int scan = strstart;
	// scanMax is the highest position that we can look at
	int scanMax = scan + std::min(DC::MAX_MATCH, lookahead) - 1;
	int limit = std::max(scan - DC::MAX_DIST, 0);
	const uint8_t *window = this->window.data();
	const int16_t *prev = this->prev.data();
	int chainLength = this->max_chain;
	int niceLength = std::min(this->niceLength, lookahead);
	matchLen = std::max(matchLen, DC::MIN_MATCH - 1);
	if (scan + matchLen > scanMax) return false;
	uint8_t scan_end1 = window[scan + matchLen - 1];
	uint8_t scan_end = window[scan + matchLen];
	// do not waste too much time if we already have a good match
	if (matchLen >= this->goodLength) chainLength >>= 2;
	do {
		match = curMatch;
		scan = strstart;
		if (window[match + matchLen] != scan_end || window[match + matchLen - 1] != scan_end1 ||
		    window[match] != window[scan] || window[++match] != window[++scan]) {
			continue;
		}
		// The reference unrolls the comparison (:510-577): (scanMax - scan) % 8 single steps, then groups of
		// 8 with the bound tested once per group.  Net effect, restated: advance while bytes agree, never
		// comparing beyond scanMax; if the byte at scanMax agrees too, scan ends at scanMax + 1.
		{
			int pre = (scanMax - scan) % 8;
			bool ok = true;
			for (int k = 0; k < pre; k++) {
				if (window[++scan] != window[++match]) { ok = false; break; }
			}
			(void)ok;
			if (window[scan] == window[match]) {
				for (;;) {
					if (scan == scanMax) {
						++scan; // advance to first position not matched
						++match;
						break;
					}
					bool all = true;
					for (int k = 0; k < 8; k++) {
						if (window[++scan] != window[++match]) { all = false; break; }
					}
					if (!all) break;
				}
			}
		}
		if (scan - strstart > matchLen) {
			matchStart = curMatch;
			matchLen = scan - strstart;
			if (matchLen >= niceLength) break;
			scan_end1 = window[scan - 1];
			scan_end = window[scan];
		}
	} while ((curMatch = (prev[curMatch & DC::WMASK] & 0xffff)) > limit && 0 != --chainLength);
	return matchLen >= DC::MIN_MATCH;
}

bool DeflaterEngine::DeflateStored(bool flush, bool finish) { // :614-649
	if (!flush && (lookahead == 0)) return false;
	strstart += lookahead;
	lookahead = 0;
	int storedLength = strstart - blockStart;
	if ((storedLength >= DC::MAX_BLOCK_SIZE) ||                         // block is full
	    (blockStart < DC::WSIZE && storedLength >= DC::MAX_DIST) ||     // block may move out of window
	    flush) {
		bool lastBlock = finish;
		if (storedLength > DC::MAX_BLOCK_SIZE) {
			storedLength = DC::MAX_BLOCK_SIZE;
			lastBlock = false;
		}
		huffman.FlushStoredBlock(window.data(), blockStart, storedLength, lastBlock);
		blockStart += storedLength;
		return !(lastBlock || storedLength == 0);
	}
	return true;
}

bool DeflaterEngine::DeflateFast(bool flush, bool finish) { // :651-739
	if (lookahead < DC::MIN_LOOKAHEAD && !flush) return false;
	while (lookahead >= DC::MIN_LOOKAHEAD || flush) {
		if (lookahead == 0) {
			// we are flushing everything
			huffman.FlushBlock(window.data(), blockStart, strstart - blockStart, finish);
			blockStart = strstart;
			return false;
		}
		if (strstart > 2 * DC::WSIZE - DC::MIN_LOOKAHEAD) {
			// slide window, as FindLongestMatch needs this
			SlideWindow();
		}
		int hashHead;
		if (lookahead >= DC::MIN_MATCH && (hashHead = InsertString()) != 0 && strategy != HuffmanOnly &&
		    strstart - hashHead <= DC::MAX_DIST && FindLongestMatch(hashHead)) {
			// longestMatch sets matchStart and matchLen
			bool full = huffman.TallyDist(strstart - matchStart, matchLen);
			lookahead -= matchLen;
			if (matchLen <= max_lazy && lookahead >= DC::MIN_MATCH) {
				while (--matchLen > 0) {
					++strstart;
					InsertString();
				}
				++strstart;
			} else {
				strstart += matchLen;
				if (lookahead >= DC::MIN_MATCH - 1) UpdateHash();
			}
			matchLen = DC::MIN_MATCH - 1;
			if (!full) continue;
		} else {
			// no match found
			huffman.TallyLit(window[strstart] & 0xff);
			++strstart;
			--lookahead;
		}
		if (huffman.IsFull()) {
			bool lastBlock = finish && (lookahead == 0);
			huffman.FlushBlock(window.data(), blockStart, strstart - blockStart, lastBlock);
			blockStart = strstart;
			return !lastBlock;
		}
	}
	return true;
}

bool DeflaterEngine::DeflateSlow(bool flush, bool finish) { // :741-855
	if (lookahead < DC::MIN_LOOKAHEAD && !flush) return false;
	while (lookahead >= DC::MIN_LOOKAHEAD || flush) {
		if (lookahead == 0) {
			if (prevAvailable) huffman.TallyLit(window[strstart - 1] & 0xff);
			prevAvailable = false;
			// we are flushing everything
			huffman.FlushBlock(window.data(), blockStart, strstart - blockStart, finish);
			blockStart = strstart;
			return false;
		}
		if (strstart >= 2 * DC::WSIZE - DC::MIN_LOOKAHEAD) {
			// slide window, as FindLongestMatch needs this
			SlideWindow();
		}
		int prevMatch = matchStart;
		int prevLen = matchLen;
		if (lookahead >= DC::MIN_MATCH) {
			int hashHead = InsertString();
			if (strategy != HuffmanOnly && hashHead != 0 && strstart - hashHead <= DC::MAX_DIST &&
			    FindLongestMatch(hashHead)) {
				// longestMatch sets matchStart and matchLen; discard match if too small and too far away
				if (matchLen <= 5 && (strategy == Filtered || (matchLen == DC::MIN_MATCH && strstart - matchStart > TooFar))) {
					matchLen = DC::MIN_MATCH - 1;
				}
			}
		}
		// previous match was better
		if ((prevLen >= DC::MIN_MATCH) && (matchLen <= prevLen)) {
			huffman.TallyDist(strstart - 1 - prevMatch, prevLen);
			prevLen -= 2;
			do {
				strstart++;
				lookahead--;
				if (lookahead >= DC::MIN_MATCH) InsertString();
			} while (--prevLen > 0);
			strstart++;
			lookahead--;
			prevAvailable = false;
			matchLen = DC::MIN_MATCH - 1;
		} else {
			if (prevAvailable) huffman.TallyLit(window[strstart - 1] & 0xff);
			prevAvailable = true;
			strstart++;
			lookahead--;
		}
		if (huffman.IsFull()) {
			int len = strstart - blockStart;
			if (prevAvailable) len--;
			bool lastBlock = (finish && (lookahead == 0) && !prevAvailable);
			huffman.FlushBlock(window.data(), blockStart, len, lastBlock);
			blockStart += len;
			return !lastBlock;
		}
	}
	return true;
}

// ============================== Zip/Compression/Deflater.cs ===============================
Deflater::Deflater(int level_, bool noZlibHeaderOrFooter_) // :178-195
	: noZlibHeaderOrFooter(noZlibHeaderOrFooter_), pending(DC::PENDING_BUF_SIZE), engine(&pending, noZlibHeaderOrFooter_) {
	level = 0; // C# field default; SetLevel(0) on a fresh object is therefore a no-op (:361), same end state
	if (level_ == -1) level_ = 6;
	else if (level_ < 0 || level_ > 9) throw SzlError(E_ARG, "level");
	SetStrategy(Default);
	SetLevel(level_);
	Reset();
}

void Deflater::Reset() { // :204-210
	state = (noZlibHeaderOrFooter ? BUSY_STATE : INIT_STATE);
	totalOut = 0;
	pending.Reset();
	engine.Reset();
}

void Deflater::SetInput(const uint8_t *input, int offset, int count) { // :331-338
	if ((state & IS_FINISHING) != 0) throw SzlError(E_STATE, "Finish() already called");
	engine.SetInput(input, offset, count);
}

void Deflater::SetLevel(int level_) { // :349-365
	if (level_ == -1) level_ = 6;
	else if (level_ < 0 || level_ > 9) throw SzlError(E_ARG, "level");
	if (level != level_) {
		level = level_;
		engine.SetLevel(level_);
	}
}

int Deflater::DeflateInto(uint8_t *output, int offset, int length) { // :427-522
	int origLength = length;
	if (state == CLOSED_STATE) throw SzlError(E_STATE, "Deflater closed");
	if (state < BUSY_STATE) {
		// output header (trap T11)
		int header = (8 + ((DC::MAX_WBITS - 8) << 4)) << 8;
		int level_flags = (level - 1) >> 1;
		if (level_flags < 0 || level_flags > 3) level_flags = 3;
		header |= level_flags << 6;
		if ((state & IS_SETDICT) != 0) header |= DC::PRESET_DICT; // dictionary was set
		header += 31 - (header % 31);
		pending.WriteShortMSB(header);
		if ((state & IS_SETDICT) != 0) {
			int chksum = engine.Adler();
			engine.ResetAdler();
			pending.WriteShortMSB(chksum >> 16);
			pending.WriteShortMSB(chksum & 0xffff);
		}
		state = BUSY_STATE | (state & (IS_FLUSHING | IS_FINISHING));
	}
	for (;;) {
		int count = pending.Flush(output, offset, length);
		offset += count;
		totalOut += count;
		length -= count;
		if (length == 0 || state == FINISHED_STATE) break;
		if (!engine.Deflate((state & IS_FLUSHING) != 0, (state & IS_FINISHING) != 0)) {
			switch (state) {
			case BUSY_STATE:
				// we need more input now
				return origLength - length;
			case FLUSHING_STATE:
				if (level != 0) {
					// supply lookahead for the inflater and fill the byte: empty static blocks (trap T6)
					int neededbits = 8 + ((-pending.BitCount()) & 7);
					while (neededbits > 0) {
						pending.WriteBits(2, 10);
						neededbits -= 10;
					}
				}
				state = BUSY_STATE;
				break;
			case FINISHING_STATE:
				pending.AlignToByte();
				// compressed data is complete; write footer information if required
				if (!noZlibHeaderOrFooter) {
					int adler = engine.Adler();
					pending.WriteShortMSB(adler >> 16);
					pending.WriteShortMSB(adler & 0xffff);
				}
				state = FINISHED_STATE;
				break;
			}
		}
	}
	return origLength - length;
}

void Deflater::SetDictionary(const uint8_t *dictionary, int index, int count) { // :559-568
	if (state != INIT_STATE) throw SzlError(E_STATE, "InvalidOperationException");
	state = SETDICT_STATE;
	engine.SetDictionary(dictionary, index, count);
}

} // namespace szl
