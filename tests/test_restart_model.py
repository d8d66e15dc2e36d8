"""CPU tier: the restart-point contract of inflate plans and the Inflater handle's algorithm over it, as a model.

`decode_slice` states what k_inflate promises for one stream of a raw plan (sharpziplib_b200/csrc/b200z_inflate.cu): decode
from bit `start_bit` of the first byte handed over, with `window` as the OutputWindow contents in front of the output;
report the output, a status, the bytes used, and the RESTART POINT = (bit, output position) of the last block header
reached.  `ModelInflater` is the handle's algorithm (b200z_handles.cu, InflaterH / inflater_run_device) transcribed: it keeps
only the input behind the restart point, the output behind min(delivered, restart point) and a 32 KiB window image, and
must deliver exactly the stream's bytes for every SetInput granularity.  The GPU tier runs the same shapes against the
real kernel and handle (tests/test_gpu_restart.py); this file pins the arithmetic (bit offsets that are not byte
aligned, window images shorter than 32 KiB, stored blocks, trailers arriving late) without a device."""
import zlib

import numpy as np
import pytest

OK, NEED, ERR = 0, 8, 3

_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
          8193, 12289, 16385, 24577]
_DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class _Short(Exception):
    pass


class _Bits:
    def __init__(self, data, pos):
        self.d, self.pos, self.n = data, pos, 8 * len(data)

    def get(self, k):
        if self.pos + k > self.n:
            raise _Short()
        v = 0
        for i in range(k):
            p = self.pos + i
            v |= ((self.d[p >> 3] >> (p & 7)) & 1) << i
        self.pos += k
        return v


def _table(lens):
    codes, code = {}, 0
    for ln in range(1, 16):
        for sym, l in enumerate(lens):
            if l == ln:
                codes[(ln, code)] = sym
                code += 1
        code <<= 1
    return codes


def _sym(br, tab):
    code = 0
    for ln in range(1, 16):
        code = (code << 1) | br.get(1)
        s = tab.get((ln, code))
        if s is not None:
            return s
    raise ValueError("bad code")


_FIXED_LIT = _table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
_FIXED_DIST = _table([5] * 32)


def decode_slice(data, start_bit=0, window=b""):
    """-> (output, status, in_used, restart_bit, restart_out)"""
    br = _Bits(data, start_bit)
    W = len(window)
    out = bytearray(window)
    rs_bit, rs_out = start_bit, 0
    good = start_bit  # bit position behind the last complete symbol / header
    last = False
    try:
        while not last:
            rs_bit, rs_out = br.pos, len(out) - W
            last = br.get(1) == 1
            btype = br.get(2)
            if btype == 0:
                br.pos = (br.pos + 7) & ~7
                ln, nl = br.get(16), br.get(16)
                if nl != ln ^ 0xFFFF:
                    return bytes(out[W:]), ERR, 0, rs_bit, rs_out
                if br.pos + 8 * ln > br.n:
                    raise _Short()  # a stored block is copied when all of it is there
                out += data[br.pos >> 3:(br.pos >> 3) + ln]
                br.pos += 8 * ln
                good = br.pos
                continue
            if btype == 1:
                lit, dist = _FIXED_LIT, _FIXED_DIST
            elif btype == 2:
                nlit, ndist, nmeta = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                ml = [0] * 19
                for i in range(nmeta):
                    ml[_ORDER[i]] = br.get(3)
                mt = _table(ml)
                lens = []
                while len(lens) < nlit + ndist:
                    s = _sym(br, mt)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.get(2))
                    elif s == 17:
                        lens += [0] * (3 + br.get(3))
                    else:
                        lens += [0] * (11 + br.get(7))
                lit, dist = _table(lens[:nlit]), _table(lens[nlit:nlit + ndist])
            else:
                return bytes(out[W:]), ERR, 0, rs_bit, rs_out
            good = br.pos
            while True:
                s = _sym(br, lit)
                if s < 256:
                    out.append(s)
                elif s == 256:
                    good = br.pos
                    break
                else:
                    ln = _LBASE[s - 257] + br.get(_LEXT[s - 257])
                    ds = _sym(br, dist)
                    d = _DBASE[ds] + br.get(_DEXT[ds])
                    for _ in range(ln):
                        out.append(out[-d] if d <= len(out) else 0)
                good = br.pos
    except _Short:
        return bytes(out[W:]), NEED, len(data), rs_bit, rs_out
    return bytes(out[W:]), OK, (good + 7) >> 3, rs_bit, rs_out


class ModelInflater:
    """InflaterH of b200z_handles.cu for raw and zlib streams (no preset dictionary)."""

    def __init__(self, raw):
        self.raw = raw
        self.input = bytearray()
        self.in_base = self.in_total = 0
        self.header_done = raw
        self.raw_off = 0
        self.rs_bit = self.rs_out = 0
        self.window = b""
        self.run_adler = 1
        self.output = bytearray()
        self.out_base = 0
        self.delivered = 0
        self.consumed = 0
        self.finished = False
        self.new_input = False
        self.runs = 0
        self.decoded_bytes = 0  # work done, to show that it is linear

    def out_total(self):
        return self.out_base + len(self.output)

    def SetInput(self, b):
        assert self.in_total <= self.consumed or self.finished
        if self.finished:
            del self.input[self.consumed - self.in_base:]
            self.in_total = self.consumed
        self.input += b
        self.in_total += len(b)
        self.new_input = True

    def _run(self):
        slice_abs = self.raw_off + (self.rs_bit >> 3)
        sbit = self.rs_bit & 7
        assert slice_abs >= self.in_base and self.in_total - slice_abs >= 0
        comp = bytes(self.input[slice_abs - self.in_base:])
        out, st, used, rbit, rout = decode_slice(comp, sbit, self.window)
        self.runs += 1
        self.decoded_bytes += len(out)
        assert st in (OK, NEED), "model streams are valid"
        del self.output[self.rs_out - self.out_base:]
        self.output += out
        if st == OK:
            self.finished = True
            self.consumed = slice_abs + used
        else:
            self.consumed = self.in_total
        assert 0 <= rout <= len(out) and sbit <= rbit <= 8 * len(comp)
        if rout > 0 or rbit != sbit:
            seg = bytes(self.output[self.rs_out - self.out_base:self.rs_out - self.out_base + rout])
            self.run_adler = zlib.adler32(seg, self.run_adler)
            self.window = (self.window + seg)[-32768:]
            self.rs_out += rout
            self.rs_bit = (self.rs_bit & ~7) + rbit
        if st == NEED:
            keep = self.raw_off + (self.rs_bit >> 3)
            if keep > self.in_base:
                del self.input[:keep - self.in_base]
                self.in_base = keep

    def Inflate(self, cap):
        if not self.finished and self.new_input:
            self.new_input = False
            if not self.header_done:
                if len(self.input) < 2:
                    self.consumed = len(self.input)
                    return b""
                assert ((self.input[0] << 8) | self.input[1]) % 31 == 0
                self.header_done = True
                self.raw_off = 2
            self._run()
            if self.finished and not self.raw:
                if self.in_total - self.consumed < 4:
                    self.finished = False
                    self.consumed = self.in_total
                else:
                    t = self.input[self.consumed - self.in_base:self.consumed - self.in_base + 4]
                    got = zlib.adler32(bytes(self.output[self.rs_out - self.out_base:]), self.run_adler)
                    assert got == int.from_bytes(t, "big"), "Adler chksum doesn't match"
                    self.adler = got
                    self.consumed += 4
        take = min(cap, self.out_total() - self.delivered)
        r = bytes(self.output[self.delivered - self.out_base:self.delivered - self.out_base + take])
        self.delivered += take
        keep = min(self.delivered, self.rs_out)
        if keep - self.out_base >= 4096:  # (the handle trims in 64 KiB steps)
            del self.output[:keep - self.out_base]
            self.out_base = keep
        return r

    @property
    def IsNeedingInput(self):
        return self.in_total <= self.consumed

    @property
    def IsFinished(self):
        return self.finished and self.delivered == self.out_total()

    @property
    def RemainingInput(self):
        return self.in_total - self.consumed


def _multi_block_stream(raw, seed=3, pieces=9):
    """text in several blocks of all three types: zlib with sync / full flushes (empty stored blocks between Huffman
    blocks, static blocks for short pieces) and a level-0 stretch"""
    rng = np.random.default_rng(seed)
    words = [bytes(rng.integers(97, 123, int(rng.integers(2, 9)), dtype=np.uint8)) for _ in range(200)]
    def text(n):
        out = bytearray()
        while len(out) < n:
            out += words[int(rng.integers(0, 200)) if rng.random() < 0.8 else int(rng.integers(0, 20))] + b" "
        return bytes(out[:n])
    co = zlib.compressobj(6, zlib.DEFLATED, -15 if raw else 15)
    orig, comp = bytearray(), bytearray()
    for i in range(pieces):
        t = text(int(rng.integers(1, 4000)))
        orig += t
        comp += co.compress(t)
        # Z_BLOCK ends the block without aligning: the next header starts inside a byte
        comp += co.flush([zlib.Z_BLOCK, zlib.Z_BLOCK, zlib.Z_SYNC_FLUSH, zlib.Z_BLOCK, zlib.Z_FULL_FLUSH][i % 5])
    noise = bytes(rng.integers(0, 256, 3000, dtype=np.uint8))  # incompressible: zlib stores it
    orig += noise
    comp += co.compress(noise)
    comp += co.flush()
    return bytes(orig), bytes(comp)


def test_decode_slice_is_an_inflater():
    for raw in (True,):
        orig, comp = _multi_block_stream(raw)
        out, st, used, rbit, rout = decode_slice(comp)
        assert st == OK and out == orig and used == len(comp)
        assert zlib.decompress(comp, -15) == orig


def test_restart_points_model():
    orig, comp = _multi_block_stream(True, seed=5)
    seen = set()
    for cut in range(1, len(comp), 37):
        out, st, used, rbit, rout = decode_slice(comp[:cut])
        assert st == NEED and orig.startswith(out) and rout <= len(out)
        seen.add(rbit & 7)
        out2, st2, used2, _, _ = decode_slice(comp[rbit >> 3:], rbit & 7, orig[max(0, rout - 32768):rout])
        assert st2 == OK and out2 == orig[rout:] and (rbit >> 3) + used2 == len(comp)
    assert len(seen - {0}) >= 3  # restart bits that are not byte aligned were exercised


@pytest.mark.parametrize("raw", [True, False])
@pytest.mark.parametrize("chunk", [1, 3, 64, 1000, 100000])
def test_handle_model_any_granularity(raw, chunk):
    orig, comp = _multi_block_stream(raw, seed=11, pieces=14 if chunk > 1 else 5)
    data = comp + b"TAIL"
    m = ModelInflater(raw)
    got = bytearray()
    pos = 0
    while not m.IsFinished:
        r = m.Inflate(777)
        got += r
        if not r and m.IsNeedingInput and not m.IsFinished:
            assert pos < len(data)
            m.SetInput(data[pos:pos + chunk])
            pos += chunk
    assert bytes(got) == orig
    assert m.consumed == len(comp) and m.RemainingInput == min(pos, len(data)) - len(comp)
    # bounded state: never more than the current block (+ what the caller has not fetched) is held
    assert len(m.input) <= len(data) and len(m.window) <= 32768
    # linear work: every run decodes on from the last block header, so a run costs at most one block (here < 4000 bytes of
    # output) on top of the new bytes, not the whole stream so far
    assert m.decoded_bytes <= len(orig) + m.runs * 4000, (m.decoded_bytes, len(orig), m.runs)
