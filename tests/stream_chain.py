"""Open runs of a level 5-9 stream chained as the Deflater handle chains them (b200z_handles.cu): every run gets the
history in front of its data (all of it in the hash chains), the stream position of its data, the sub-byte tail of the
output so far and the parse state the previous run stopped in; the next run starts at the cut the previous one reported.
`runner` runs one segment -- the CPU model or a device plan -- so both tiers share the bookkeeping."""
import zlib

CLEAN = (0, 2, 0)


class Chain:
    def __init__(self, runner, dictionary=None):
        """runner(hist, mask, seg, pos_base, bit_base, end_mode, entry) -> (bytes, nbits, (covered, next_entry) or None);
        mask flags the history positions that never went into the hash chains (the last two of a dictionary)"""
        self.runner = runner
        self.hist = bytearray()
        self.mask = bytearray()
        self.seen = 0
        self.tail_bits = self.tail_count = 0
        self.out = bytearray()
        self.entry = CLEAN
        self.adler = 1
        self.log = []  # per run: (bytes handed to it, bits written, covered, entry of the next run)
        self.end_bits = []  # per run: the bit position in .out where its output ends
        if dictionary is not None and len(dictionary) >= 3:
            self._remember(dictionary[-32506:], 2)

    def _remember(self, seg, uninserted=0):
        self.hist += seg
        self.mask += bytes(max(0, len(seg) - uninserted)) + b"\1" * min(uninserted, len(seg))
        cut = max(0, len(self.hist) - 32768)
        del self.hist[:cut]
        del self.mask[:cut]
        self.seen += len(seg)

    def run(self, seg, end_mode):
        o, nb, cut = self.runner(bytes(self.hist), bytes(self.mask), seg, self.seen, self.tail_count, end_mode, self.entry)
        o = bytearray(o[:(nb + 7) // 8])
        if o:
            o[0] |= self.tail_bits
        whole = nb // 8
        self.out += o[:whole]
        self.tail_count = nb & 7
        self.tail_bits = (o[whole] & ((1 << self.tail_count) - 1)) if self.tail_count else 0
        if end_mode in (0, 1) and self.tail_count:  # the stream ends: AlignToByte (Deflater.cs:507)
            self.out.append(self.tail_bits)
            self.tail_bits = self.tail_count = 0
        self.end_bits.append(8 * len(self.out) + self.tail_count)
        covered, nxt = cut if end_mode == 3 else (len(seg), CLEAN)
        self.log.append((len(seg), nb, covered, nxt))
        self.adler = zlib.adler32(bytes(seg[:covered]), self.adler)
        self._remember(seg[:covered])
        self.entry = nxt
        return covered

    def finish_after_flush(self):
        # Finish() behind a completed Flush(): the empty final static block (value 3 in 10 bits), then byte alignment
        v = self.tail_bits | (3 << self.tail_count)
        n = self.tail_count + 10
        while n > 0:
            self.out.append(v & 0xFF)
            v >>= 8
            n -= 8
        self.tail_bits = self.tail_count = 0


def chained(runner, data, run_lens, close, dictionary=None):
    """Open runs of run_lens[i] new bytes each (plus what the run in front left behind its cut), then everything left in
    one closing run: close 0 Finish, 1 Flush then Finish, 2 Flush followed by Finish() with nothing new.  Returns the
    chain (raw deflate bytes in .out, running Adler-32 of the data in .adler)."""
    ch = Chain(runner, dictionary)
    pos, carried = 0, 0
    for L in run_lens:
        seg = data[pos:pos + carried + L]
        covered = ch.run(seg, 3)
        pos += covered
        carried = len(seg) - covered
    ch.run(data[pos:], close)
    if close == 2:
        ch.finish_after_flush()
    return ch


def random_runs(rnd, n, lo, hi):
    """run lengths drawn from [lo, hi) that leave between 0 and hi bytes for the closing run"""
    out, left = [], n
    while left > 2 * hi:
        L = rnd.randrange(lo, hi)
        out.append(L)
        left -= L
    return out


def zlib_frame(level, raw, adler, dictionary=None):
    """the zlib framing the handle writes (Deflater.cs:436-464 header, DICTID, Adler-32 trailer)"""
    header = (8 + (7 << 4)) << 8
    lf = (level - 1) >> 1
    header |= (lf if 0 <= lf <= 3 else 3) << 6
    if dictionary is not None:
        header |= 0x20
    header += 31 - header % 31
    h = bytes([header >> 8, header & 0xFF])
    if dictionary is not None:
        h += zlib.adler32(dictionary).to_bytes(4, "big")
    return h + bytes(raw) + adler.to_bytes(4, "big")
