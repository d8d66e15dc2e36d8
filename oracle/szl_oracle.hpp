// szl_oracle.hpp -- CPU parity ORACLE for the SharpZipLib DEFLATE hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under sharpziplib_b200/ (the product) may
// include, link or call this.  Only tests/, __graft_entry__.smoke() and the
// cpu_baseline / --impl reference legs of bench.py use it, as the checker / CPU
// baseline.
//
// This is a single-threaded C++17 restatement of the reference's managed C#
// algorithm (ICSharpCode.SharpZipLib v1.4.2), following the reference's control
// flow and variable names so it can be audited side by side.  Paths below are
// relative to SharpZipLib's src/ICSharpCode.SharpZipLib/.
//
// Pinning status (see DESIGN.md "Oracle"):
//   * Crc32 / Adler32  : PINNED by the reference's known-answer tests
//                        (test/.../Checksum/ChecksumTests.cs:24-37,107-146).
//   * Inflater         : PINNED by the reference's foreign-compressor fixtures
//                        (test/.../Zip/ZipCorruptionHandling.cs:12-69) and by
//                        agreement with zlib on valid streams.
//   * Deflater bytes   : PINNED IN PART.  The reference tree holds two raw deflate streams its own Deflater
//                        wrote: the payload inside the AES-encrypted archive of
//                        test/.../Zip/ZipEncryptionHandling.cs:452-456 (a DYNAMIC block for 56 bytes of text --
//                        zlib emits a static block for that input at every level, SharpZipLib's tree
//                        construction and block decision do not) and the entry of TestFileBadCDGoodCD64.
//                        Both are reproduced byte for byte at levels 1-9 (tests/test_oracle.py
//                        test_deflater_bytes_against_streams_the_reference_holds): that pins Tree.BuildTree /
//                        BuildLength / BuildCodes, SendAllTrees / WriteTree, FlushBlock's decision,
//                        CompressBlock and the bit writer.  Neither input has a repeated trigram, so the
//                        match finding (FindLongestMatch / DeflateSlow / DeflateFast) is PARITY UNPINNED:
//                        no .NET runtime exists here or on the GPU boxes, and those bytes rest on the audit
//                        of this restatement against the cited lines plus structural checks (every output
//                        inflates to its input under zlib; feed-pattern invariance; debug invariants).
#pragma once
#include <cstdint>
#include <cstddef>
#include <stdexcept>
#include <string>
#include <vector>

namespace szl {

// ---- error model: .NET exception classes mapped to a code (SURVEY 8b) -------------------
enum ErrKind : int {
	E_OK = 0,
	E_ARG = 1,     // ArgumentNullException / ArgumentOutOfRangeException / ArgumentException
	E_STATE = 2,   // InvalidOperationException
	E_DATA = 3,    // SharpZipBaseException / StreamDecodingException / ValueOutOfRangeException
	E_INTERNAL = 4 // IndexOutOfRangeException etc. (e.g. PendingBuffer overflow, trap T12)
};

struct SzlError : public std::runtime_error {
	int kind;
	SzlError(int k, const std::string &m) : std::runtime_error(m), kind(k) {}
};

// ---- Checksum/Adler32.cs, Checksum/Crc32.cs, Checksum/CrcUtilities.cs -------------------
class Adler32 {
public:
	Adler32() { Reset(); }
	void Reset() { checkValue = 1; }                      // Adler32.cs:76-79
	uint32_t Value() const { return checkValue; }         // Adler32.cs:84-90
	void HarnessSetValue(uint32_t v) { checkValue = v; }  // harness-only (no reference counterpart)
	void Update(int bval);                                // Adler32.cs:96-108
	void Update(const uint8_t *buf, size_t off, size_t count); // Adler32.cs:134-161
private:
	uint32_t checkValue;
};

class Crc32 {
public:
	Crc32() { Reset(); }
	void Reset() { checkValue = 0xFFFFFFFFu; }            // Crc32.cs:75-78
	uint32_t Value() const { return checkValue ^ 0xFFFFFFFFu; } // Crc32.cs:85-91
	void HarnessSetValue(uint32_t v) { checkValue = v ^ 0xFFFFFFFFu; } // harness-only (no reference counterpart)
	void Update(int bval);                                // Crc32.cs:100-103
	void Update(const uint8_t *buf, size_t off, size_t count); // Crc32.cs:138-159
private:
	uint32_t checkValue;
};

// ---- Zip/Compression/PendingBuffer.cs + DeflaterPending.cs ------------------------------
class PendingBuffer {
public:
	explicit PendingBuffer(int bufferSize) : buffer(bufferSize), start(0), end(0), bits(0), bitCount(0) {}
	void Reset() { start = end = bitCount = 0; }          // PendingBuffer.cs:53-56 (bits NOT cleared)
	void WriteByte(int value) { put((uint8_t)value); }
	void WriteShort(int value) { put((uint8_t)value); put((uint8_t)(value >> 8)); }
	void WriteBlock(const uint8_t *block, int offset, int length);
	int BitCount() const { return bitCount; }
	void AlignToByte();                                   // PendingBuffer.cs:143-161
	void WriteBits(int b, int count);                     // PendingBuffer.cs:168-189
	void WriteShortMSB(int s) { put((uint8_t)(s >> 8)); put((uint8_t)s); }
	bool IsFlushed() const { return end == 0; }
	int Flush(uint8_t *output, int offset, int length);   // PendingBuffer.cs:226-248
private:
	void put(uint8_t v) {
		if (end >= (int)buffer.size()) throw SzlError(E_INTERNAL, "PendingBuffer overflow (IndexOutOfRangeException)");
		buffer[end++] = v;
	}
	std::vector<uint8_t> buffer;
	int start, end;
	uint32_t bits;
	int bitCount;
};

enum DeflateStrategy { Default = 0, Filtered = 1, HuffmanOnly = 2 };

// ---- Zip/Compression/DeflaterHuffman.cs --------------------------------------------------
class DeflaterHuffman {
public:
	explicit DeflaterHuffman(PendingBuffer *pending);
	void Reset();
	void FlushStoredBlock(const uint8_t *stored, int storedOffset, int storedLength, bool lastBlock);
	void FlushBlock(const uint8_t *stored, int storedOffset, int storedLength, bool lastBlock);
	bool IsFull() const { return last_lit >= BUFSIZE; }
	bool TallyLit(int literal);
	bool TallyDist(int distance, int length);
	static int16_t BitReverse(int toReverse);

	// instrumentation for tests (not part of the reference surface)
	struct BlockTrace { int type; int nsyms; int storedLength; int opt_len; int static_len; };
	std::vector<BlockTrace> *trace = nullptr;

	static constexpr int BUFSIZE = 1 << (8 + 6);
	static constexpr int LITERAL_NUM = 286;
	static constexpr int DIST_NUM = 30;
	static constexpr int BITLEN_NUM = 19;

	struct Tree {
		std::vector<int16_t> freqs;
		std::vector<uint8_t> length;
		bool haveLength = false;
		int minNumCodes;
		int numCodes = 0;
		std::vector<int16_t> codes;
		std::vector<int> bl_counts;
		int maxLength;
		DeflaterHuffman *dh;
		Tree(DeflaterHuffman *dh_, int elems, int minCodes, int maxLength_);
		void Reset();
		void WriteSymbol(int code);
		void SetStaticCodes(const int16_t *staticCodes, const uint8_t *staticLengths, int n);
		void BuildCodes();
		void BuildTree();
		int GetEncodedLength() const;
		void CalcBLFreq(Tree &blTree);
		void WriteTree(Tree &blTree);
		void BuildLength(const std::vector<int> &childs);
	};

	PendingBuffer *pending;
	Tree literalTree, distTree, blTree;
	std::vector<int16_t> d_buf;
	std::vector<uint8_t> l_buf;
	int last_lit = 0;
	int extra_bits = 0;

private:
	void SendAllTrees(int blTreeCodes);
	void CompressBlock();
	static int Lcode(int length);
	static int Dcode(int distance);
};

// ---- Zip/Compression/DeflaterEngine.cs ---------------------------------------------------
class DeflaterEngine {
public:
	DeflaterEngine(PendingBuffer *pending, bool noAdlerCalculation);
	bool Deflate(bool flush, bool finish);
	void SetInput(const uint8_t *buffer, int offset, int count);
	bool NeedsInput() const { return inputEnd == inputOff; }
	void SetDictionary(const uint8_t *buffer, int offset, int length);
	void Reset();
	void ResetAdler() { if (hasAdler) adler.Reset(); }
	int Adler() const { return hasAdler ? (int)adler.Value() : 0; }
	int64_t TotalIn() const { return totalIn; }
	DeflateStrategy strategy = Default;
	void SetLevel(int level);
	void FillWindow();
	DeflaterHuffman huffman;

private:
	void UpdateHash();
	int InsertString();
	void SlideWindow();
	bool FindLongestMatch(int curMatch);
	bool DeflateStored(bool flush, bool finish);
	bool DeflateFast(bool flush, bool finish);
	bool DeflateSlow(bool flush, bool finish);

	int ins_h = 0;
	std::vector<int16_t> head, prev;
	int matchStart = 0, matchLen = 0;
	bool prevAvailable = false;
	int blockStart, strstart, lookahead = 0;
	std::vector<uint8_t> window;
	int max_chain = 0, max_lazy = 0, niceLength = 0, goodLength = 0;
	int compressionFunction = 0;
	const uint8_t *inputBuf = nullptr;
	int64_t totalIn = 0;
	int inputOff = 0, inputEnd = 0;
	PendingBuffer *pending;
	bool hasAdler;
	Adler32 adler;
};

// ---- Zip/Compression/Deflater.cs ---------------------------------------------------------
class Deflater {
public:
	Deflater(int level, bool noZlibHeaderOrFooter);
	void Reset();
	int Adler() const { return engine.Adler(); }
	int64_t TotalIn() const { return engine.TotalIn(); }
	int64_t TotalOut() const { return totalOut; }
	void Flush() { state |= IS_FLUSHING; }
	void Finish() { state |= (IS_FLUSHING | IS_FINISHING); }
	bool IsFinished() const { return state == FINISHED_STATE && pending.IsFlushed(); }
	bool IsNeedingInput() const { return engine.NeedsInput(); }
	void SetInput(const uint8_t *input, int offset, int count);
	void SetLevel(int level);
	int GetLevel() const { return level; }
	void SetStrategy(DeflateStrategy s) { engine.strategy = s; }
	int DeflateInto(uint8_t *output, int offset, int length);
	void SetDictionary(const uint8_t *dict, int index, int count);
	DeflaterEngine &Engine() { return engine; }

private:
	static constexpr int IS_SETDICT = 0x01, IS_FLUSHING = 0x04, IS_FINISHING = 0x08;
	static constexpr int INIT_STATE = 0x00, SETDICT_STATE = 0x01, BUSY_STATE = 0x10, FLUSHING_STATE = 0x14,
	                     FINISHING_STATE = 0x1c, FINISHED_STATE = 0x1e, CLOSED_STATE = 0x7f;
	int level = -2; // the C# field defaults to 0; see ctor note in the .cpp
	bool noZlibHeaderOrFooter;
	int state = 0;
	int64_t totalOut = 0;
	PendingBuffer pending;
	DeflaterEngine engine;
};

// ---- Zip/Compression/Streams/StreamManipulator.cs ----------------------------------------
class StreamManipulator {
public:
	int PeekBits(int bitCount);
	bool TryGetBits(int bitCount, int &output, int outputOffset = 0);
	bool TryGetBits(int bitCount, uint8_t *array, int index);
	void DropBits(int bitCount) { buffer_ >>= bitCount; bitsInBuffer_ -= bitCount; }
	int AvailableBits() const { return bitsInBuffer_; }
	int AvailableBytes() const { return windowEnd_ - windowStart_ + (bitsInBuffer_ >> 3); }
	void SkipToByteBoundary() { buffer_ >>= (bitsInBuffer_ & 7); bitsInBuffer_ &= ~7; }
	bool IsNeedingInput() const { return windowStart_ == windowEnd_; }
	int CopyBytes(uint8_t *output, int offset, int length);
	void Reset() { buffer_ = 0; windowStart_ = windowEnd_ = bitsInBuffer_ = 0; }
	void SetInput(const uint8_t *buffer, int offset, int count);
private:
	const uint8_t *window_ = nullptr;
	int windowStart_ = 0, windowEnd_ = 0;
	uint32_t buffer_ = 0;
	int bitsInBuffer_ = 0;
};

// ---- Zip/Compression/Streams/OutputWindow.cs ---------------------------------------------
class OutputWindow {
public:
	OutputWindow() : window(WindowSize, 0) {}
	void Write(int value);
	void Repeat(int length, int distance);
	int CopyStored(StreamManipulator &input, int length);
	void CopyDict(const uint8_t *dictionary, int offset, int length);
	int GetFreeSpace() const { return WindowSize - windowFilled; }
	int GetAvailable() const { return windowFilled; }
	int CopyOutput(uint8_t *output, int offset, int len);
	void Reset() { windowFilled = windowEnd = 0; }
private:
	static constexpr int WindowSize = 1 << 15, WindowMask = WindowSize - 1;
	void SlowRepeat(int repStart, int length, int distance);
	std::vector<uint8_t> window;
	int windowEnd = 0, windowFilled = 0;
};

// ---- Zip/Compression/InflaterHuffmanTree.cs ----------------------------------------------
class InflaterHuffmanTree {
public:
	InflaterHuffmanTree(const uint8_t *codeLengths, int count) { BuildTree(codeLengths, count); }
	int GetSymbol(StreamManipulator &input);
	static InflaterHuffmanTree &defLitLenTree();
	static InflaterHuffmanTree &defDistTree();
private:
	void BuildTree(const uint8_t *codeLengths, int count);
	std::vector<int16_t> tree;
	int16_t at(int idx) const {
		if (idx < 0 || idx >= (int)tree.size()) throw SzlError(E_INTERNAL, "InflaterHuffmanTree index out of range");
		return tree[idx];
	}
};

// ---- Zip/Compression/InflaterDynHeader.cs ------------------------------------------------
class InflaterDynHeader {
public:
	explicit InflaterDynHeader(StreamManipulator *input_) : input(input_) {}
	~InflaterDynHeader();
	bool AttemptRead();
	InflaterHuffmanTree *TakeLiteralLengthTree();
	InflaterHuffmanTree *TakeDistanceTree();
private:
	bool Step(bool &current); // one MoveNext of the C# iterator
	StreamManipulator *input;
	int pc = 0; // resume point of the iterator
	bool done = false, lastCurrent = false;
	uint8_t codeLengths[286 + 30] = {0};
	InflaterHuffmanTree *metaCodeTree = nullptr, *litLenTree = nullptr, *distTree = nullptr;
	int litLenCodeCount = 0, distanceCodeCount = 0, metaCodeCount = 0;
	int dataCodeCount = 0, i = 0, index = 0, symbol = 0, repeatCount = 0;
	uint8_t codeLength = 0;
};

// ---- Zip/Compression/Inflater.cs ---------------------------------------------------------
class Inflater {
public:
	explicit Inflater(bool noHeader);
	~Inflater();
	void Reset();
	void SetDictionary(const uint8_t *buffer, int index, int count);
	void SetInput(const uint8_t *buffer, int index, int count);
	int Inflate(uint8_t *buffer, int bufferLength, int offset, int count);
	bool IsNeedingInput() const { return input.IsNeedingInput(); }
	bool IsNeedingDictionary() const { return mode == DECODE_DICT && neededBits == 0; }
	bool IsFinished() const { return mode == FINISHED && outputWindow.GetAvailable() == 0; }
	int Adler() const;
	int64_t TotalOut() const { return totalOut; }
	int64_t TotalIn() const { return totalIn - (int64_t)RemainingInput(); }
	int RemainingInput() const { return input.AvailableBytes(); }
private:
	enum {
		DECODE_HEADER = 0, DECODE_DICT = 1, DECODE_BLOCKS = 2, DECODE_STORED_LEN1 = 3, DECODE_STORED_LEN2 = 4,
		DECODE_STORED = 5, DECODE_DYN_HEADER = 6, DECODE_HUFFMAN = 7, DECODE_HUFFMAN_LENBITS = 8,
		DECODE_HUFFMAN_DIST = 9, DECODE_HUFFMAN_DISTBITS = 10, DECODE_CHKSUM = 11, FINISHED = 12
	};
	bool DecodeHeader();
	bool DecodeDict();
	bool DecodeHuffman();
	bool DecodeChksum();
	bool Decode();
	void dropTrees();
	int mode;
	int readAdler = 0, neededBits = 0, repLength = 0, repDist = 0, uncomprLen = 0;
	bool isLastBlock = false;
	int64_t totalOut = 0, totalIn = 0;
	bool noHeader;
	StreamManipulator input;
	OutputWindow outputWindow;
	InflaterDynHeader *dynHeader = nullptr;
	InflaterHuffmanTree *litlenTree = nullptr, *distTree = nullptr;
	bool treesOwned = false;
	bool hasAdler;
	Adler32 adler;
};

} // namespace szl
