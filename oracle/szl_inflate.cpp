// szl_inflate.cpp -- ORACLE (test infrastructure): Inflater side.
// Restates Zip/Compression/{Inflater,InflaterDynHeader,InflaterHuffmanTree}.cs and
// Zip/Compression/Streams/{OutputWindow,StreamManipulator}.cs of the reference (paths relative
// to SharpZipLib's src/ICSharpCode.SharpZipLib/).  See szl_oracle.hpp for the pinning status.
#include "szl_oracle.hpp"
#include <algorithm>
#include <cstring>

namespace szl {

// ============================== Streams/StreamManipulator.cs ==============================
int StreamManipulator::PeekBits(int bitCount) { // :31-44
	if (bitsInBuffer_ < bitCount) {
		if (windowStart_ == windowEnd_) return -1; // ok
		uint32_t lo = window_[windowStart_++] & 0xffu;
		uint32_t hi = window_[windowStart_++] & 0xffu;
		buffer_ |= (uint32_t)((lo | (hi << 8)) << bitsInBuffer_);
		bitsInBuffer_ += 16;
	}
	return (int)(buffer_ & (uint32_t)((1 << bitCount) - 1));
}

bool StreamManipulator::TryGetBits(int bitCount, int &output, int outputOffset) { // :53-63
	int bits = PeekBits(bitCount);
	if (bits < 0) return false;
	output = bits + outputOffset;
	DropBits(bitCount);
	return true;
}

bool StreamManipulator::TryGetBits(int bitCount, uint8_t *array, int index) { // :72-82
	int bits = PeekBits(bitCount);
	if (bits < 0) return false;
	array[index] = (uint8_t)bits;
	DropBits(bitCount);
	return true;
}

int StreamManipulator::CopyBytes(uint8_t *output, int offset, int length) { // :183-227
	if (length < 0) throw SzlError(E_ARG, "length");
	if ((bitsInBuffer_ & 7) != 0) throw SzlError(E_STATE, "Bit buffer is not byte aligned!");
	int count = 0;
	while ((bitsInBuffer_ > 0) && (length > 0)) {
		output[offset++] = (uint8_t)buffer_;
		buffer_ >>= 8;
		bitsInBuffer_ -= 8;
		length--;
		count++;
	}
	if (length == 0) return count;
	int avail = windowEnd_ - windowStart_;
	if (length > avail) length = avail;
	std::memcpy(output + offset, window_ + windowStart_, (size_t)length);
	windowStart_ += length;
	if (((windowStart_ - windowEnd_) & 1) != 0) {
		// we always want an even number of bytes in input, see PeekBits
		buffer_ = (uint32_t)(window_[windowStart_++] & 0xff);
		bitsInBuffer_ = 8;
	}
	return count + length;
}

void StreamManipulator::SetInput(const uint8_t *buffer, int offset, int count) { // :244-289
	if (buffer == nullptr) throw SzlError(E_ARG, "buffer");
	if (offset < 0) throw SzlError(E_ARG, "offset Cannot be negative");
	if (count < 0) throw SzlError(E_ARG, "count Cannot be negative");
	if (windowStart_ < windowEnd_) throw SzlError(E_STATE, "Old input was not completely processed");
	int end = offset + count;
	if (offset > end) throw SzlError(E_ARG, "count");
	if ((count & 1) != 0) {
		// we always want an even number of bytes in input, see PeekBits
		buffer_ |= (uint32_t)((buffer[offset++] & 0xff) << bitsInBuffer_);
		bitsInBuffer_ += 8;
	}
	window_ = buffer;
	windowStart_ = offset;
	windowEnd_ = end;
}

// ============================== Streams/OutputWindow.cs ===================================
void OutputWindow::Write(int value) { // :35-43
	if (windowFilled++ == WindowSize) throw SzlError(E_STATE, "Window full");
	window[windowEnd++] = (uint8_t)value;
	windowEnd &= WindowMask;
}

void OutputWindow::SlowRepeat(int repStart, int length, int /*distance*/) { // :45-53
	while (length-- > 0) {
		window[windowEnd++] = window[repStart++];
		windowEnd &= WindowMask;
		repStart &= WindowMask;
	}
}

void OutputWindow::Repeat(int length, int distance) { // :63-92
	if ((windowFilled += length) > WindowSize) throw SzlError(E_STATE, "Window full");
	int repStart = (windowEnd - distance) & WindowMask;
	int border = WindowSize - length;
	if ((repStart <= border) && (windowEnd < border)) {
		if (length <= distance) {
			std::memmove(&window[windowEnd], &window[repStart], (size_t)length);
			windowEnd += length;
		} else {
			// copy manually, since the repeat pattern overlaps
			while (length-- > 0) window[windowEnd++] = window[repStart++];
		}
	} else {
		SlowRepeat(repStart, length, distance);
	}
}

int OutputWindow::CopyStored(StreamManipulator &input, int length) { // :100-122
	length = std::min(std::min(length, WindowSize - windowFilled), input.AvailableBytes());
	int copied;
	int tailLen = WindowSize - windowEnd;
	if (length > tailLen) {
		copied = input.CopyBytes(window.data(), windowEnd, tailLen);
		if (copied == tailLen) copied += input.CopyBytes(window.data(), 0, length - tailLen);
	} else {
		copied = input.CopyBytes(window.data(), windowEnd, length);
	}
	windowEnd = (windowEnd + copied) & WindowMask;
	windowFilled += copied;
	return copied;
}

void OutputWindow::CopyDict(const uint8_t *dictionary, int offset, int length) { // :133-153
	if (dictionary == nullptr) throw SzlError(E_ARG, "dictionary");
	if (windowFilled > 0) throw SzlError(E_STATE, "InvalidOperationException");
	if (length > WindowSize) {
		offset += length - WindowSize;
		length = WindowSize;
	}
	std::memcpy(window.data(), dictionary + offset, (size_t)length);
	windowEnd = length & WindowMask;
}

int OutputWindow::CopyOutput(uint8_t *output, int offset, int len) { // :182-209
	int copyEnd = windowEnd;
	if (len > windowFilled) len = windowFilled;
	else copyEnd = (windowEnd - windowFilled + len) & WindowMask;
	int copied = len;
	int tailLen = len - copyEnd;
	if (tailLen > 0) {
		std::memcpy(output + offset, &window[WindowSize - tailLen], (size_t)tailLen);
		offset += tailLen;
		len = copyEnd;
	}
	std::memcpy(output + offset, &window[copyEnd - len], (size_t)len);
	windowFilled -= copied;
	if (windowFilled < 0) throw SzlError(E_STATE, "InvalidOperationException");
	return copied;
}

// ============================== InflaterHuffmanTree.cs ====================================
static int revbits(int v) { return DeflaterHuffman::BitReverse(v) & 0xffff; }

InflaterHuffmanTree &InflaterHuffmanTree::defLitLenTree() { // static ctor :34-70
	static InflaterHuffmanTree *t = [] {
		uint8_t codeLengths[288];
		int i = 0;
		while (i < 144) codeLengths[i++] = 8;
		while (i < 256) codeLengths[i++] = 9;
		while (i < 280) codeLengths[i++] = 7;
		while (i < 288) codeLengths[i++] = 8;
		return new InflaterHuffmanTree(codeLengths, 288);
	}();
	return *t;
}

InflaterHuffmanTree &InflaterHuffmanTree::defDistTree() {
	static InflaterHuffmanTree *t = [] {
		uint8_t codeLengths[32];
		for (int i = 0; i < 32; i++) codeLengths[i] = 5;
		return new InflaterHuffmanTree(codeLengths, 32);
	}();
	return *t;
}

void InflaterHuffmanTree::BuildTree(const uint8_t *codeLengths, int count) { // :87-169
	const int MAX_BITLEN = 15;
	int blCount[MAX_BITLEN + 1] = {0};
	int nextCode[MAX_BITLEN + 1] = {0};
	for (int i = 0; i < count; i++) {
		int bits = codeLengths[i];
		if (bits > 0) blCount[bits]++;
	}
	int code = 0;
	int treeSize = 512;
	for (int bits = 1; bits <= MAX_BITLEN; bits++) {
		nextCode[bits] = code;
		code += blCount[bits] << (16 - bits);
		if (bits >= 10) {
			// an extra table is needed for bit lengths >= 10
			int start = nextCode[bits] & 0x1ff80;
			int end = code & 0x1ff80;
			treeSize += (end - start) >> (16 - bits);
		}
	}
	// (the completeness check "code != 65536" is commented out in the reference, :116-121, trap T13)
	if (treeSize < 512) treeSize = 512; // .NET would throw on a negative array size; never reached for sane input
	tree.assign((size_t)treeSize, 0);
	int treePtr = 512;
	for (int bits = MAX_BITLEN; bits >= 10; bits--) {
		int end = code & 0x1ff80;
		code -= blCount[bits] << (16 - bits);
		int start = code & 0x1ff80;
		for (int i = start; i < end; i += 1 << 7) {
			int idx = revbits(i);
			if (idx >= (int)tree.size()) throw SzlError(E_INTERNAL, "InflaterHuffmanTree build index out of range");
			tree[idx] = (int16_t)((-treePtr << 4) | bits);
			treePtr += 1 << (bits - 9);
		}
	}
	for (int i = 0; i < count; i++) {
		int bits = codeLengths[i];
		if (bits == 0) continue;
		code = nextCode[bits];
		int revcode = revbits(code);
		if (bits <= 9) {
			do {
				if (revcode >= (int)tree.size()) throw SzlError(E_INTERNAL, "InflaterHuffmanTree build index out of range");
				tree[revcode] = (int16_t)((i << 4) | bits);
				revcode += 1 << bits;
			} while (revcode < 512);
		} else {
			int subTree = at(revcode & 511);
			int treeLen = 1 << (subTree & 15);
			subTree = -(subTree >> 4);
			do {
				int idx = subTree | (revcode >> 9);
				if (idx < 0 || idx >= (int)tree.size()) throw SzlError(E_INTERNAL, "InflaterHuffmanTree build index out of range");
				tree[idx] = (int16_t)((i << 4) | bits);
				revcode += 1 << bits;
			} while (revcode < treeLen);
		}
		nextCode[bits] = code + (1 << (16 - bits));
	}
}

int InflaterHuffmanTree::GetSymbol(StreamManipulator &input) { // :181-235
	int lookahead, symbol;
	if ((lookahead = input.PeekBits(9)) >= 0) {
		symbol = at(lookahead);
		int bitlen = symbol & 15;
		if (symbol >= 0) {
			if (bitlen == 0) throw SzlError(E_DATA, "Encountered invalid codelength 0");
			input.DropBits(bitlen);
			return symbol >> 4;
		}
		int subtree = -(symbol >> 4);
		if ((lookahead = input.PeekBits(bitlen)) >= 0) {
			symbol = at(subtree | (lookahead >> 9));
			input.DropBits(symbol & 15);
			return symbol >> 4;
		} else {
			int bits = input.AvailableBits();
			lookahead = input.PeekBits(bits);
			symbol = at(subtree | (lookahead >> 9));
			if ((symbol & 15) <= bits) {
				input.DropBits(symbol & 15);
				return symbol >> 4;
			} else {
				return -1;
			}
		}
	} else { // less than 9 bits
		int bits = input.AvailableBits();
		lookahead = input.PeekBits(bits);
		symbol = at(lookahead);
		if (symbol >= 0 && (symbol & 15) <= bits) {
			input.DropBits(symbol & 15);
			return symbol >> 4;
		} else {
			return -1;
		}
	}
}

// ============================== InflaterDynHeader.cs ======================================
static const int MetaCodeLengthIndex[] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15}; // :24-25

InflaterDynHeader::~InflaterDynHeader() {
	delete metaCodeTree;
	delete litLenTree;
	delete distTree;
}

bool InflaterDynHeader::AttemptRead() { // :32-33  "!state.MoveNext() || state.Current"
	if (done) return true; // MoveNext() is false after the iterator completed
	bool current = false;
	bool moved = Step(current);
	if (!moved) return true;
	return current;
}

InflaterHuffmanTree *InflaterDynHeader::TakeLiteralLengthTree() { // :122-123
	if (!litLenTree) throw SzlError(E_DATA, "Header properties were accessed before header had been successfully read");
	InflaterHuffmanTree *t = litLenTree;
	litLenTree = nullptr;
	return t;
}

InflaterHuffmanTree *InflaterDynHeader::TakeDistanceTree() { // :128-129
	if (!distTree) throw SzlError(E_DATA, "Header properties were accessed before header had been successfully read");
	InflaterHuffmanTree *t = distTree;
	distTree = nullptr;
	return t;
}

// One MoveNext() of the C# iterator CreateStateMachine (:42-120).  Returns false when the iterator has
// completed; otherwise sets `current` to the yielded value.  `pc` records the yield point to resume at.
bool InflaterDynHeader::Step(bool &current) {
	switch (pc) {
	case 0: break;
	case 1: goto L1;
	case 2: goto L2;
	case 3: goto L3;
	case 4: goto L4;
	case 5: goto L5;
	case 6: goto L6;
	case 7: goto L7;
	case 8: goto L8;
	case 9: done = true; return false; // resumed after the final "yield return true": iterator ends
	default: done = true; return false;
	}
	// read initial code length counts from header
L1:
	if (!input->TryGetBits(5, litLenCodeCount, 257)) { pc = 1; current = false; return true; }
L2:
	if (!input->TryGetBits(5, distanceCodeCount, 1)) { pc = 2; current = false; return true; }
L3:
	if (!input->TryGetBits(4, metaCodeCount, 4)) { pc = 3; current = false; return true; }
	dataCodeCount = litLenCodeCount + distanceCodeCount;
	if (litLenCodeCount > 286) throw SzlError(E_DATA, "ValueOutOfRangeException: litLenCodeCount");
	if (distanceCodeCount > 30) throw SzlError(E_DATA, "ValueOutOfRangeException: distanceCodeCount");
	if (metaCodeCount > 19) throw SzlError(E_DATA, "ValueOutOfRangeException: metaCodeCount");
	// load code lengths for the meta tree from the header bits
	for (i = 0; i < metaCodeCount; i++) {
	L4:
		if (!input->TryGetBits(3, codeLengths, MetaCodeLengthIndex[i])) { pc = 4; current = false; return true; }
	}
	// (the reference passes the whole 316-entry codeLengths array as the meta tree's lengths, :67)
	metaCodeTree = new InflaterHuffmanTree(codeLengths, 286 + 30);
	// decompress the meta tree symbols into the data table code lengths
	index = 0;
	while (index < dataCodeCount) {
	L5:
		if ((symbol = metaCodeTree->GetSymbol(*input)) < 0) { pc = 5; current = false; return true; }
		if (symbol < 16) {
			// append literal code length
			codeLengths[index++] = (uint8_t)symbol;
		} else {
			repeatCount = 0;
			if (symbol == 16) { // repeat last code length 3..6 times
				if (index == 0)
					throw SzlError(E_DATA, "Cannot repeat previous code length when no other code length has been read");
				codeLength = codeLengths[index - 1];
			L6:
				if (!input->TryGetBits(2, repeatCount, 3)) { pc = 6; current = false; return true; }
			} else if (symbol == 17) { // repeat zero 3..10 times
				codeLength = 0;
			L7:
				if (!input->TryGetBits(3, repeatCount, 3)) { pc = 7; current = false; return true; }
			} else { // (symbol == 18), repeat zero 11..138 times
				codeLength = 0;
			L8:
				if (!input->TryGetBits(7, repeatCount, 11)) { pc = 8; current = false; return true; }
			}
			if (index + repeatCount > dataCodeCount)
				throw SzlError(E_DATA, "Cannot repeat code lengths past total number of data code lengths");
			while (repeatCount-- > 0) codeLengths[index++] = codeLength;
		}
	}
	if (codeLengths[256] == 0) throw SzlError(E_DATA, "Inflater dynamic header end-of-block code missing");
	litLenTree = new InflaterHuffmanTree(codeLengths, litLenCodeCount);
	distTree = new InflaterHuffmanTree(codeLengths + litLenCodeCount, distanceCodeCount);
	pc = 9;
	current = true;
	return true;
}

// ============================== Inflater.cs ===============================================
static const int CPLENS[] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258}; // :39-42
static const int CPLEXT[] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};                             // :47-50
static const int CPDIST[] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577}; // :55-59
static const int CPDEXT[] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};                   // :64-68

Inflater::Inflater(bool noHeader_) : noHeader(noHeader_), hasAdler(!noHeader_) { // :172-180
	mode = noHeader ? DECODE_BLOCKS : DECODE_HEADER;
}

Inflater::~Inflater() {
	dropTrees();
	delete dynHeader;
}

void Inflater::dropTrees() {
	if (treesOwned) {
		delete litlenTree;
		delete distTree;
	}
	litlenTree = distTree = nullptr;
	treesOwned = false;
}

void Inflater::Reset() { // :188-200
	mode = noHeader ? DECODE_BLOCKS : DECODE_HEADER;
	totalIn = 0;
	totalOut = 0;
	input.Reset();
	outputWindow.Reset();
	delete dynHeader;
	dynHeader = nullptr;
	dropTrees();
	isLastBlock = false;
	if (hasAdler) adler.Reset();
}

bool Inflater::DecodeHeader() { // :209-250
	int header = input.PeekBits(16);
	if (header < 0) return false;
	input.DropBits(16);
	// the header is written in "wrong" byte order
	header = ((header << 8) | (header >> 8)) & 0xffff;
	if (header % 31 != 0) throw SzlError(E_DATA, "Header checksum illegal");
	if ((header & 0x0f00) != (8 << 8)) throw SzlError(E_DATA, "Compression Method unknown");
	if ((header & 0x0020) == 0) { // dictionary flag?
		mode = DECODE_BLOCKS;
	} else {
		mode = DECODE_DICT;
		neededBits = 32;
	}
	return true;
}

bool Inflater::DecodeDict() { // :258-272
	while (neededBits > 0) {
		int dictByte = input.PeekBits(8);
		if (dictByte < 0) return false;
		input.DropBits(8);
		readAdler = (int)(((uint32_t)readAdler << 8) | (uint32_t)dictByte);
		neededBits -= 8;
	}
	return false;
}

bool Inflater::DecodeHuffman() { // :283-386
	int free = outputWindow.GetFreeSpace();
	while (free >= 258) {
		int symbol;
		switch (mode) {
		case DECODE_HUFFMAN:
			// this is the inner loop
			while (((symbol = litlenTree->GetSymbol(input)) & ~0xff) == 0) {
				outputWindow.Write(symbol);
				if (--free < 258) return true;
			}
			if (symbol < 257) {
				if (symbol < 0) return false;
				// symbol == 256: end of block
				dropTrees();
				mode = DECODE_BLOCKS;
				return true;
			}
			if (symbol - 257 >= (int)(sizeof(CPLENS) / sizeof(CPLENS[0]))) throw SzlError(E_DATA, "Illegal rep length code");
			repLength = CPLENS[symbol - 257];
			neededBits = CPLEXT[symbol - 257];
			/* fall through */
		case DECODE_HUFFMAN_LENBITS:
			if (neededBits > 0) {
				mode = DECODE_HUFFMAN_LENBITS;
				int i = input.PeekBits(neededBits);
				if (i < 0) return false;
				input.DropBits(neededBits);
				repLength += i;
			}
			mode = DECODE_HUFFMAN_DIST;
			/* fall through */
		case DECODE_HUFFMAN_DIST:
			symbol = distTree->GetSymbol(input);
			if (symbol < 0) return false;
			if (symbol >= (int)(sizeof(CPDIST) / sizeof(CPDIST[0]))) throw SzlError(E_DATA, "Illegal rep dist code");
			repDist = CPDIST[symbol];
			neededBits = CPDEXT[symbol];
			/* fall through */
		case DECODE_HUFFMAN_DISTBITS:
			if (neededBits > 0) {
				mode = DECODE_HUFFMAN_DISTBITS;
				int i = input.PeekBits(neededBits);
				if (i < 0) return false;
				input.DropBits(neededBits);
				repDist += i;
			}
			outputWindow.Repeat(repLength, repDist);
			free -= repLength;
			mode = DECODE_HUFFMAN;
			break;
		default: throw SzlError(E_DATA, "Inflater unknown mode");
		}
	}
	return true;
}

bool Inflater::DecodeChksum() { // :397-418
	while (neededBits > 0) {
		int chkByte = input.PeekBits(8);
		if (chkByte < 0) return false;
		input.DropBits(8);
		readAdler = (int)(((uint32_t)readAdler << 8) | (uint32_t)chkByte);
		neededBits -= 8;
	}
	if ((int)adler.Value() != readAdler) throw SzlError(E_DATA, "Adler chksum doesn't match");
	mode = FINISHED;
	return false;
}

bool Inflater::Decode() { // :429-552
	switch (mode) {
	case DECODE_HEADER: return DecodeHeader();
	case DECODE_DICT: return DecodeDict();
	case DECODE_CHKSUM: return DecodeChksum();
	case DECODE_BLOCKS: {
		if (isLastBlock) {
			if (noHeader) {
				mode = FINISHED;
				return false;
			} else {
				input.SkipToByteBoundary();
				neededBits = 32;
				mode = DECODE_CHKSUM;
				return true;
			}
		}
		int type = input.PeekBits(3);
		if (type < 0) return false;
		input.DropBits(3);
		isLastBlock |= (type & 1) != 0;
		switch (type >> 1) {
		case 0: // STORED_BLOCK
			input.SkipToByteBoundary();
			mode = DECODE_STORED_LEN1;
			break;
		case 1: // STATIC_TREES
			dropTrees();
			litlenTree = &InflaterHuffmanTree::defLitLenTree();
			distTree = &InflaterHuffmanTree::defDistTree();
			treesOwned = false;
			mode = DECODE_HUFFMAN;
			break;
		case 2: // DYN_TREES
			delete dynHeader;
			dynHeader = new InflaterDynHeader(&input);
			mode = DECODE_DYN_HEADER;
			break;
		default: throw SzlError(E_DATA, "Unknown block type");
		}
		return true;
	}
	case DECODE_STORED_LEN1:
		if ((uncomprLen = input.PeekBits(16)) < 0) return false;
		input.DropBits(16);
		mode = DECODE_STORED_LEN2;
		/* fall through */
	case DECODE_STORED_LEN2: {
		int nlen = input.PeekBits(16);
		if (nlen < 0) return false;
		input.DropBits(16);
		if (nlen != (uncomprLen ^ 0xffff)) throw SzlError(E_DATA, "broken uncompressed block");
		mode = DECODE_STORED;
	}
		/* fall through */
	case DECODE_STORED: {
		int more = outputWindow.CopyStored(input, uncomprLen);
		uncomprLen -= more;
		if (uncomprLen == 0) {
			mode = DECODE_BLOCKS;
			return true;
		}
		return !input.IsNeedingInput();
	}
	case DECODE_DYN_HEADER:
		if (!dynHeader->AttemptRead()) return false;
		dropTrees();
		litlenTree = dynHeader->TakeLiteralLengthTree();
		distTree = dynHeader->TakeDistanceTree();
		treesOwned = true;
		mode = DECODE_HUFFMAN;
		/* fall through */
	case DECODE_HUFFMAN:
	case DECODE_HUFFMAN_LENBITS:
	case DECODE_HUFFMAN_DIST:
	case DECODE_HUFFMAN_DISTBITS: return DecodeHuffman();
	case FINISHED: return false;
	default: throw SzlError(E_DATA, "Inflater.Decode unknown mode");
	}
}

void Inflater::SetDictionary(const uint8_t *buffer, int index, int count) { // :589-620
	if (buffer == nullptr) throw SzlError(E_ARG, "buffer");
	if (index < 0) throw SzlError(E_ARG, "index");
	if (count < 0) throw SzlError(E_ARG, "count");
	if (!IsNeedingDictionary()) throw SzlError(E_STATE, "Dictionary is not needed");
	if (hasAdler) adler.Update(buffer, (size_t)index, (size_t)count);
	if (hasAdler && (int)adler.Value() != readAdler) throw SzlError(E_DATA, "Wrong adler checksum");
	if (hasAdler) adler.Reset();
	outputWindow.CopyDict(buffer, index, count);
	mode = DECODE_BLOCKS;
}

void Inflater::SetInput(const uint8_t *buffer, int index, int count) { // :653-657
	input.SetInput(buffer, index, count);
	totalIn += (int64_t)count;
}

int Inflater::Inflate(uint8_t *buffer, int bufferLength, int offset, int count) { // :715-777
	if (buffer == nullptr) throw SzlError(E_ARG, "buffer");
	if (count < 0) throw SzlError(E_ARG, "count cannot be negative");
	if (offset < 0) throw SzlError(E_ARG, "offset cannot be negative");
	if (offset + count > bufferLength) throw SzlError(E_ARG, "count exceeds buffer bounds");
	// special case: count may be zero
	if (count == 0) {
		if (!IsFinished()) Decode(); // -jr- 08-Nov-2003 INFLATE_BUG fix..
		return 0;
	}
	int bytesCopied = 0;
	do {
		if (mode != DECODE_CHKSUM) {
			// don't give away any output, if we are waiting for the checksum in the input stream
			int more = outputWindow.CopyOutput(buffer, offset, count);
			if (more > 0) {
				if (hasAdler) adler.Update(buffer, (size_t)offset, (size_t)more);
				offset += more;
				bytesCopied += more;
				totalOut += (int64_t)more;
				count -= more;
				if (count == 0) return bytesCopied;
			}
		}
	} while (Decode() || ((outputWindow.GetAvailable() > 0) && (mode != DECODE_CHKSUM)));
	return bytesCopied;
}

int Inflater::Adler() const { // :823-842
	if (IsNeedingDictionary()) return readAdler;
	else if (hasAdler) return (int)adler.Value();
	else return 0;
}

} // namespace szl
