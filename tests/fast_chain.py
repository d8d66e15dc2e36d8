"""Open runs of a level 0-4 stream chained as the Deflater handle chains them (b200z_handles.cu): every run gets the last
32768 bytes in front of its data as history, the stream position of its data, the sub-byte tail of the output so far, the
engine state the previous run left (a flush, or the cut of an open run) and its SetInput calls; the next run starts at the
cut the previous one reported, with the rest of the call the cut fell into as its first call.  `runner` runs one
segment -- the CPU model or a device plan -- so both tiers share the bookkeeping."""
import struct
import zlib

FAST_STATE_BYTES = 2 * 65536 + 64
STORED_STATE_BYTES = 16


def new_state(level):
    return bytes(STORED_STATE_BYTES if level == 0 else FAST_STATE_BYTES)


def handed(level, state, covered):
    """data bytes of the run that the engine's window held at its cut: strstart - blockStart at level 0, the lookahead at
    levels 1-4 (strstart == blockStart there)"""
    if level == 0:
        strstart, block_start = struct.unpack_from("<ii", state, 0)
        return covered + strstart - block_start
    return covered + struct.unpack_from("<i", state, 131072 + 8)[0]


def live_state(level, state):
    """the part of an engine state that a run reads for certain: DeflateStored's fields; DeflateFast's head[] and scalars.
    prev[] is left out: in the slots of positions that DeflateFast never inserted (inside a match longer than max_lazy) the
    serial engine keeps what was there, k_fast's group step the link it wrote up front, and no chain walk reads either"""
    return state if level == 0 else state[:65536] + state[131072:]


def live_log(level, log):
    return [e[:5] + (live_state(level, e[5]),) for e in log]


def shift_position(level, state, k):
    """the same engine k * 32768 stream bytes later: slides + k, input_off + 32768 k (mod 2^32, as the fields hold it)"""
    b = bytearray(state)
    off = 8 if level == 0 else 131072 + 24
    slides, inp = struct.unpack_from("<II", b, off)
    struct.pack_into("<II", b, off, (slides + k) & 0xFFFFFFFF, (inp + 32768 * k) & 0xFFFFFFFF)
    return bytes(b)


class FastChain:
    def __init__(self, runner, level, dictionary=None):
        """runner(hist, seg, pos_base, bit_base, calls, end_mode, state, cont) -> (bytes, nbits, (covered, call), state);
        (covered, call) only for END_NONE runs, covered 0 when no block closed (the state is then what it was)"""
        self.runner = runner
        self.level = level
        self.hist = bytearray()
        self.seen = 0
        self.started = False
        self.state = new_state(level)
        self.tail_bits = self.tail_count = 0
        self.out = bytearray()
        self.adler = 1
        self.log = []  # per run: (bytes, calls, bits written, covered, call, state after it)
        self.end_bits = []  # per run: the bit position in .out where its output ends
        # per open run that closed a block: (stream offset of the run's data, covered, [start, end) of the call of the cut in
        # the run's data, data bytes the window had taken at the cut)
        self.cuts = []
        if dictionary is not None and len(dictionary) >= 3:
            self._remember(dictionary[-32506:])

    def _remember(self, seg):
        self.hist += seg
        del self.hist[:max(0, len(self.hist) - 32768)]
        self.seen += len(seg)

    def run(self, seg, calls, end_mode):
        assert sum(calls) == len(seg)
        bit_base = self.tail_count
        o, nb, cut, state = self.runner(bytes(self.hist), bytes(seg), self.seen, self.tail_count, list(calls), end_mode,
                                        self.state, self.started)
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
        covered, call = cut if end_mode == 3 else (len(seg), None)
        self.log.append((len(seg), tuple(calls), nb, covered, call, state))
        if end_mode == 3 and covered == 0:
            assert nb == bit_base
            return 0, None
        if end_mode == 3:
            start = sum(calls[:call])
            self.cuts.append((self.seen, covered, (start, start + calls[call]), handed(self.level, state, covered)))
        self.state = state
        self.started = True
        self.adler = zlib.adler32(bytes(seg[:covered]), self.adler)
        self._remember(seg[:covered])
        return covered, call

    def finish_after_flush(self):
        # Finish() behind a completed Flush(): the empty final block -- static (value 3 in 10 bits) at levels 1-4, an
        # empty stored block at level 0 -- then byte alignment
        if self.level == 0:
            self.out += bytes([1, 0, 0, 0xFF, 0xFF])
            return
        v = self.tail_bits | (3 << self.tail_count)
        n = self.tail_count + 10
        while n > 0:
            self.out.append(v & 0xFF)
            v >>= 8
            n -= 8
        self.tail_bits = self.tail_count = 0


def chained(runner, level, data, calls, run_lens, close, dictionary=None):
    """Open runs that take the SetInput calls in front of them (behind what the previous run carried) while they add at
    most run_lens[i] bytes, at least one call; then everything left in one closing run: close 0 Finish, 1 Flush then
    Finish, 2 Flush followed by Finish() with nothing new.  Returns the chain (raw deflate bytes in .out, running Adler-32
    of the data in .adler)."""
    ch = FastChain(runner, level, dictionary)
    pos, k = 0, 0
    pend = []  # the calls the last run carried: the rest of the call of its cut, then the ones behind it
    for L in run_lens:
        run_calls = list(pend)
        carried = sum(pend)
        add = 0
        while k < len(calls) and (add == 0 or add + calls[k] <= L):
            run_calls.append(calls[k])
            add += calls[k]
            k += 1
        if not add:
            break
        seg = data[pos:pos + carried + add]
        covered, call = ch.run(seg, run_calls, 3)
        if covered:
            end = sum(run_calls[:call + 1])
            pend = [end - covered] + run_calls[call + 1:]
            pos += covered
        else:
            pend = run_calls
    ch.run(data[pos:], pend + list(calls[k:]), close)
    if close == 2:
        ch.finish_after_flush()
    return ch
