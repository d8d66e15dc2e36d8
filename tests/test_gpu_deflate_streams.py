"""GPU tier: Deflater sets (b200z_deflate_streams_*, DeflaterSet).  Every stream's output is compared with the oracle's
Deflater fed the same SetInput / drain / Flush / Finish calls, with a Deflater handle fed the same calls, and with zlib /
gzip inflating it back.  Tests named *small* also run on the CUDA emulator (tests/test_deflate_streams_emu.py), which builds
the library with a smaller open-run size and says so in B200Z_SET_RUN_BYTES."""
import os
import random
import struct
import zlib

import numpy as np
import pytest

from sharpziplib_b200 import _lib, datagen

pytestmark = pytest.mark.gpu

K = int(os.environ.get("B200Z_SET_RUN_BYTES", 4456448))  # kSetRunBytes of the library under test
GZ_HEADER = bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF])
WRAPS = [_lib.WRAP_RAW, _lib.WRAP_ZLIB, _lib.WRAP_GZIP, _lib.WRAP_RAW_CRC32]


class Reference:
    """one stream as the reference writes it: oracle Deflater behind DeflaterOutputStream (GZipOutputStream for gzip)"""

    def __init__(self, oracle, level, strategy, wrap):
        self.d = oracle.Deflater(level, nowrap=wrap != _lib.WRAP_ZLIB)
        self.d.set_strategy(strategy)
        self.wrap = wrap
        self.out = bytearray(GZ_HEADER if wrap == _lib.WRAP_GZIP else b"")
        self.data = bytearray()

    def _drain(self):
        while True:
            b = self.d.deflate(65536)
            if not b:
                break
            self.out += b

    def write(self, buf, op):
        self.d.set_input(buf)
        self.data += buf
        if len(buf):
            self._drain()
        if op == 1:
            self.d.flush()
            self._drain()
        elif op == 2:
            self.d.finish()
            self._drain()
            if self.wrap == _lib.WRAP_GZIP:
                self.out += struct.pack("<II", zlib.crc32(bytes(self.data)), len(self.data) & 0xFFFFFFFF)


class Handle:
    """the same calls on a Deflater handle (raw or zlib: the body of every wrap)"""

    def __init__(self, z, level, strategy, wrap):
        self.d = z.Deflater(level, wrap != _lib.WRAP_ZLIB)
        self.d.SetStrategy(strategy)
        self.out = bytearray()
        self.buf = bytearray(1 << 20)

    def _drain(self):
        while True:
            k = self.d.Deflate(self.buf)
            if k <= 0:
                break
            self.out += self.buf[:k]

    def write(self, buf, op):
        self.d.SetInput(buf)
        while not self.d.IsNeedingInput:
            self._drain()
        if op:
            self.d.Flush() if op == 1 else self.d.Finish()
            self._drain()


def body(out, wrap):
    return out[10:-8] if wrap == _lib.WRAP_GZIP else out


def corpus(seed, n):
    """random bytes and text in 8 KiB pieces: blocks close well inside any open run, at every level"""
    rng = np.random.default_rng(seed)
    text = datagen.silesia_mix(seed, n, config=3)
    out = np.empty(n, np.uint8)
    for a in range(0, n, 16384):
        out[a:a + 8192] = rng.integers(0, 256, min(8192, n - a), dtype=np.uint8)
        out[a + 8192:a + 16384] = text[a + 8192:a + 16384]
    return out.tobytes()


def pieces(rnd, data, sizes):
    out, pos = [], 0
    while pos < len(data):
        c = min(rnd.choice(sizes), len(data) - pos)
        out.append(data[pos:pos + c])
        pos += c
    return out


def run_script(z, oracle, level, strategy, wrap, streams, ops_of, handles=True):
    """streams finish in different calls: stream i finishes right behind its last write"""
    n = len(streams)
    s = z.DeflaterSet(n, level=level, strategy=strategy, wrap=wrap)
    refs = [Reference(oracle, level, strategy, wrap) for _ in range(n)]
    hs = [Handle(z, level, strategy, wrap) for _ in range(n)] if handles else []
    got = [bytearray() for _ in range(n)]
    n_calls = max(len(w) for w in streams) + 1
    done = [False] * n
    for k in range(n_calls):
        bufs, ops = [], []
        for i, w in enumerate(streams):
            if k < len(w):
                bufs.append(w[k])
                ops.append(ops_of(i, k))
            elif k == len(w):
                bufs.append(b"")
                ops.append(2)
            else:
                bufs.append(b"")
                ops.append(0)
        s.write(bufs, ops)  # (a finished stream stays in with an empty write and op 0: no call)
        assert not s.status.any()
        for i, part in enumerate(s.read()):
            got[i] += part
        for i in range(n):
            if done[i]:
                continue
            refs[i].write(bufs[i], ops[i])
            if hs:
                hs[i].write(bufs[i], ops[i])
            done[i] = ops[i] == 2
    checks = s.checks()
    stats = s.stats()
    s.close()
    for i in range(n):
        data = bytes(refs[i].data)
        assert bytes(got[i]) == bytes(refs[i].out), (level, strategy, wrap, i)
        if hs:
            assert body(bytes(got[i]), wrap) == bytes(hs[i].out), (level, strategy, wrap, i)
        if wrap == _lib.WRAP_ZLIB:
            assert zlib.decompress(bytes(got[i])) == data and checks[i] == zlib.adler32(data)
        elif wrap == _lib.WRAP_GZIP:
            assert zlib.decompress(bytes(got[i]), 31) == data and checks[i] == zlib.crc32(data)
        else:
            assert zlib.decompress(bytes(got[i]), -15) == data
            assert checks[i] == (zlib.crc32(data) if wrap == _lib.WRAP_RAW_CRC32 else 0)
    return stats


# ---- small: also on the emulator -----------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [0, 1, 6])
def test_small_three_streams_two_open_runs(z, oracle, level):
    """three streams written in pieces across the slide point; two of them pass through two open runs, one flushes"""
    rnd = random.Random(level)
    sizes = [0, 1, 4093, 65273, 65274, 65275, K // 3]
    streams = [pieces(rnd, corpus(10 + i, int(2.6 * K) if i < 2 else K // 2), sizes) for i in range(3)]
    stats = run_script(z, oracle, level, 0, _lib.WRAP_ZLIB, streams, lambda i, k: 1 if (i == 2 and k % 3 == 1) else 0)
    assert stats["runs"] >= 4 + 3 and stats["held"] <= 2 * K + 2 * (K // 3)


@pytest.mark.parametrize("level", [0, 2, 3, 4, 6])
def test_small_stream_starts_next_to_continuing_ones(z, oracle, level):
    """a stream's first segment in the same plan as streams that already ran: it continues from nothing (no history, the
    fresh engine state), for a flush, a finish and an open run"""
    a, b, c = corpus(21, 70000), corpus(22, 50000), corpus(23, 40000)
    d, e = corpus(24, int(1.05 * K)), corpus(25, int(1.05 * K))
    streams = [[a[:30000], a[30000:], e],  # flushes in calls 0 and 1, then an open run next to stream 3's first
               [b"", b[:20000], b[20000:]],  # starts in call 1 and flushes there
               [b"", c],                     # starts in call 1 and finishes in call 2
               [b"", b"", d]]                # starts with an open run in call 2
    ops = {(0, 0): 1, (0, 1): 1, (1, 1): 1}
    run_script(z, oracle, level, 0, _lib.WRAP_ZLIB, streams, lambda i, k: ops.get((i, k), 0))


# ---- GPU only ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", range(10))
def test_levels_wraps_strategies(z, oracle, level):
    rnd = random.Random(100 + level)
    for wrap in WRAPS:
        for strategy in range(3):
            streams = [pieces(rnd, corpus(rnd.randrange(1 << 30), n), [0, 1, 4093, 30000, 65274, 65275, 70000])
                       for n in (150000, 90000, 3)]
            run_script(z, oracle, level, strategy, wrap, streams,
                       lambda i, k: 1 if (i == 0 and k % 4 == 2) or (i == 1 and k == 1) else 0)


@pytest.mark.parametrize("n", [1, 2, 37, 1024])
def test_many_streams(z, oracle, n):
    rnd = random.Random(n)
    streams = [pieces(rnd, corpus(i, rnd.choice([0, 1, 5000, 40000, 140000])), [0, 1, 4093, 20000, 65274])
               for i in range(n)]
    for level in ((1, 6) if n < 1024 else (6,)):
        run_script(z, oracle, level, 0, _lib.WRAP_GZIP if n == 37 else _lib.WRAP_ZLIB, streams,
                   lambda i, k: 1 if (i % 3 == 0 and k % 2 == 1) else 0, handles=n < 1024)


@pytest.mark.parametrize("level", [1, 4, 6, 9])
def test_long_streams_through_several_open_runs(z, oracle, level):
    """three streams of more than 3 x kSetRunBytes in 1 MiB writes, next to a short one; the bytes held stay bounded"""
    log = datagen.log_stream(int(3.3 * K), config=4).tobytes()
    mix = corpus(7, int(3.5 * K))
    rnd = random.Random(level)
    streams = [pieces(rnd, log, [1 << 20]), pieces(rnd, mix, [1 << 20, 65274, 4093]), pieces(rnd, mix[::-1], [1 << 20]),
               [b"short"]]
    stats = run_script(z, oracle, level, 0, _lib.WRAP_ZLIB, streams, lambda i, k: 1 if (i == 1 and k == 5) else 0)
    assert stats["runs"] >= 3 * 2 + 4  # (levels 0-4 end runs at a write: 1 MiB writes make them about 5 MiB long)
    assert stats["held"] <= 2 * K + 2 * (1 << 20), stats


def test_finished_stream_refuses_more_input_alone(z, oracle):
    s = z.DeflaterSet(3, level=6)
    a, b = corpus(1, 50000), corpus(2, 60000)
    s.write([a, b, b""], [2, 0, 0])
    s.write([b"", b, b""], [0, 0, 0])  # nothing for the finished stream: no call, no error
    assert not s.status.any()
    with pytest.raises(z.InvalidOperationException):
        s.write([b"more", b"", b"x"], [0, 2, 2])
    assert list(s.status) == [_lib.E_STATE, _lib.OK, _lib.OK]
    for op in (1, 2):
        with pytest.raises(z.InvalidOperationException):
            s.write([b"", b"", b""], [op, 0, 0])
        assert list(s.status) == [_lib.E_STATE, _lib.OK, _lib.OK]
    out = s.read()
    assert zlib.decompress(out[0]) == a and zlib.decompress(out[1]) == b + b and zlib.decompress(out[2]) == b"x"
    assert s.stats()["plans"] == 2
    s.close()


def test_open_runs_of_many_streams_split_by_plan_bytes(z, oracle):
    """240 streams due for an open run in one call, more than 1 GiB together: the set splits them into plans of at most
    1 GiB of input, so one plan's workspace does not grow with the number of streams"""
    n, size = 240, K + 300000
    base = corpus(31, size + n * 4096)
    streams = [base[i * 4096:i * 4096 + size] for i in range(n)]
    s = z.DeflaterSet(n, level=1)
    s.write(streams, [0] * n)
    first = s.stats()
    s.write([b""] * n, [2] * n)
    out = s.read()
    st = s.stats()
    s.close()
    assert first["runs"] == n and first["plans"] == 2, first
    assert 0 < st["workspace"] < 20 << 30, st
    for i in range(n):
        assert zlib.decompress(out[i]) == streams[i]
    for i in (0, n - 1):
        r = Reference(oracle, 1, 0, _lib.WRAP_ZLIB)
        r.write(streams[i], 2)
        assert out[i] == bytes(r.out)


def test_arguments_and_refusals(z):
    with pytest.raises(ValueError):
        z.DeflaterSet(2, level=10)
    with pytest.raises(ValueError):
        z.DeflaterSet(2, wrap=4)
    s = z.DeflaterSet(2, level=-1)
    with pytest.raises(ValueError):
        s.write([b"a", b"b"], [0, 3])
    assert s.read() == [b"", b""]
    s.close()
    with pytest.raises(z.B200zUnsupported):
        z.deflate_batch([b"abc" * 1000], level=6, end_mode=_lib.END_NONE)
    with pytest.raises(z.B200zUnsupported):
        z.Pipeline.deflate([3000], level=6, end_mode=_lib.END_NONE)
