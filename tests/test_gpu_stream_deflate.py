"""GPU tier: open runs of levels 5-9 (B200Z_END_NONE), by hand through the plan calls and inside the Deflater handle.
Tests named *small* also run on the CUDA emulator (tests/test_stream_deflate.py)."""
import random
import time
import zlib

import numpy as np
import pytest

from sharpziplib_b200 import _lib
from stream_chain import CLEAN, chained, random_runs, zlib_frame

pytestmark = pytest.mark.gpu


def plan_runner(z, level, strategy, pos_shift=0):
    """one run as a single-stream device plan: history in front of the data, entry state set, cut read back"""
    import torch

    def run(hist, mask, seg, pos_base, bit_base, end_mode, entry):
        p = z.DeflatePlan([len(seg)], level=level, strategy=strategy, end_mode=end_mode,
                          history=([len(hist)], [pos_base + pos_shift], [bit_base], [mask]), entry=[entry])
        hin = np.zeros(p.in_bytes, np.uint8)
        o = int(p.in_offsets[0])
        blob = np.frombuffer(hist + bytes(seg), np.uint8)
        hin[o:o + blob.size] = blob
        di = torch.from_numpy(hin).cuda()
        do = torch.zeros(p.out_bytes, dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_st = torch.zeros(1, dtype=torch.int32, device="cuda")
        d_bits = torch.zeros(1, dtype=torch.int64, device="cuda")
        p.run(di, do, d_len, d_st, None, d_bits)
        torch.cuda.synchronize()
        assert int(d_st.cpu()[0]) == 0
        nb = int(d_bits.cpu()[0])
        oo = int(p.out_offsets[0])
        out = do.cpu().numpy()[oo:oo + (nb + 7) // 8].tobytes()
        cut = None
        if end_mode == _lib.END_NONE:
            cov, ents = p.cut()
            cut = (int(cov[0]), tuple(int(x) for x in ents[0]))
        p.close()
        return out, nb, cut
    return run


def stream_corpus():
    from test_stream_deflate import stream_corpus as c
    return c()


# ---- small: also on the emulator -----------------------------------------------------------------------------------
def small_data():
    rng = np.random.default_rng(11)
    from sharpziplib_b200 import datagen
    return (rng.integers(0, 256, 40000, dtype=np.uint8).tobytes() + datagen.silesia_mix(0, 30000, config=9).tobytes()
            + rng.integers(0, 256, 20000, dtype=np.uint8).tobytes())


@pytest.mark.parametrize("level", [6, 9])
def test_small_open_runs_match_oracle(z, oracle, level):
    data = small_data()
    for close in (0, 1):
        ch = chained(plan_runner(z, level, 0), data, [25000, 20000], close)
        assert bytes(ch.out) == oracle.deflate(data, level=level, pattern=close)
        assert all(c > 0 for (_, _, c, _) in ch.log[:-1])


def test_small_open_runs_refused_where_no_cut_can_be_returned(z):
    for level in (0, 1, 4):
        with pytest.raises(z.B200zUnsupported):
            z.DeflatePlan([100000], level=level, end_mode=_lib.END_NONE)
    with pytest.raises(z.B200zUnsupported):
        z.deflate_batch([b"abc" * 1000], level=6, end_mode=_lib.END_NONE)
    with pytest.raises(z.B200zUnsupported):
        z.Pipeline.deflate([3000], level=6, end_mode=_lib.END_NONE)
    p = z.DeflatePlan([1000], level=6)
    with pytest.raises(z.InvalidOperationException):
        p.cut()
    with pytest.raises(ValueError):  # a pending match needs a pending byte
        p.set_entry([(0, 5, 10)])


# ---- plan level ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [5, 6, 7, 8, 9])
def test_open_runs_chained_by_hand(z, oracle, level):
    data = stream_corpus()
    rnd = random.Random(100 + level)
    for strategy in (0, 1, 2):
        want = {p: oracle.deflate(data, level=level, strategy=strategy, pattern=p) for p in (0, 1)}
        for close in (0, 1, 2):
            ch = chained(plan_runner(z, level, strategy), data, random_runs(rnd, len(data), 4_000_000, 5_000_000), close)
            assert bytes(ch.out) == want[0 if close == 0 else 1], (strategy, close)
            if close == 0:
                zl = oracle.deflate(data, level=level, nowrap=False, strategy=strategy)
                assert zlib_frame(level, ch.out, ch.adler) == zl


def test_open_runs_equal_cpu_model(z):
    """covered bytes, bit lengths and entry states of every run are the CPU model's"""
    from test_stream_deflate import model_lib, model_runner
    M = model_lib()
    data = stream_corpus()
    runs = random_runs(random.Random(5), len(data), 4_000_000, 5_000_000)
    for level, strategy in ((6, 0), (9, 1)):
        a = chained(plan_runner(z, level, strategy), data, runs, 2)
        b = chained(model_runner(M, level, strategy), data, runs, 2)
        assert a.log == b.log


def test_open_runs_after_dictionary(z, oracle):
    from helpers import oracle_calls
    data = stream_corpus()[:13_000_000]
    dictionary = data[5_000_000:5_040_000]
    ch = chained(plan_runner(z, 6, 0), data, [4_200_000, 4_700_000], 0, dictionary=dictionary)
    assert zlib_frame(6, ch.out, ch.adler, dictionary) == oracle_calls(6, [(data, [len(data)])], dictionary=dictionary)


def test_position_beyond_4gib_is_the_same_phase(z):
    """a run at stream position P and at P + k * 32768 > 2^32 writes the same bytes (stored blocks and slide positions
    depend on the phase only)"""
    rng = np.random.default_rng(3)
    data = rng.integers(0, 256, 1_500_000, dtype=np.uint8).tobytes() + stream_corpus()[:3_000_000]
    hist = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    P = 100000
    k = (2 ** 32 - P) // 32768 + 1
    assert P + k * 32768 > 2 ** 32
    for end_mode in (_lib.END_NONE, _lib.END_FINISH):
        for level in (6, 9):
            a = plan_runner(z, level, 0)(hist, bytes(32768), data, P, 3, end_mode, CLEAN)
            b = plan_runner(z, level, 0, pos_shift=k * 32768)(hist, bytes(32768), data, P, 3, end_mode, CLEAN)
            assert a == b, (end_mode, level)


# ---- the Deflater handle -------------------------------------------------------------------------------------------
class _Sink:
    def __init__(self, keep=True):
        self.keep = keep
        self.buf = bytearray()
        self.n = 0

    def write(self, b):
        self.n += len(b)
        if self.keep:
            self.buf += b


@pytest.mark.parametrize("level", [6, 9])
def test_handle_600mib_with_a_flush(z, oracle, level):
    from helpers import oracle_calls
    from sharpziplib_b200 import datagen
    rng = np.random.default_rng(level)
    base = datagen.log_stream(200 << 20)
    mixed = np.concatenate([base, rng.integers(0, 256, 40 << 20, dtype=np.uint8), base[::-1].copy(),
                            base[:160 << 20]]).tobytes()
    half = 330 << 20
    sink = _Sink()
    s = z.DeflaterOutputStream(sink, z.Deflater(level))
    rnd = random.Random(level)
    pos, flushed, total_out_before = 0, False, 0
    while pos < len(mixed):
        step = rnd.choice([1, 4097, 65536, 1 << 20, 3 << 20, 7 << 20])
        if not flushed and pos + step > half:
            step = half - pos
        s.Write(mixed[pos:pos + step])
        pos += step
        if pos == half and not flushed:
            s.Flush()
            flushed = True
    total_out_before = s.deflater_.TotalOut
    s.Finish()
    assert total_out_before > 0
    want = oracle_calls(level, [(mixed[:half], [half]), (mixed[half:], [len(mixed) - half])], nowrap=False)
    assert bytes(sink.buf) == want
    assert s.deflater_.TotalIn == len(mixed)
    assert s.deflater_.Adler == zlib.adler32(mixed)


def test_gzip_stream_over_4gib(z):
    """about 4.5 GiB of log lines through GZipOutputStream in 1 MiB writes: inflates back (CRC-32 and length of the
    output equal the input's), ISIZE = TotalIn mod 2^32"""
    from sharpziplib_b200 import datagen
    pool = datagen.log_stream(96 << 20).tobytes()
    total = (9 << 29) + 12345  # 4.5 GiB + a little

    class Check:
        def __init__(self):
            self.d = zlib.decompressobj(31)
            self.crc = 0
            self.n = 0
            self.tail = b""
            self.comp = 0

        def write(self, b):
            self.comp += len(b)
            out = self.d.decompress(b)
            self.crc = zlib.crc32(out, self.crc)
            self.n += len(out)
            self.tail = (self.tail + bytes(b))[-8:]

    ck = Check()
    g = z.GZipOutputStream(ck)
    g.ModifiedTime = 0
    t0 = time.time()
    crc, pos, k = 0, 0, 0
    while pos < total:
        off = (k * 7919 * 4096) % (len(pool) - (1 << 20))
        m = min(1 << 20, total - pos)
        piece = pool[off:off + m]
        crc = zlib.crc32(piece, crc)
        g.Write(piece)
        pos += m
        k += 1
    g.Finish()
    secs = time.time() - t0
    ck.d.flush()
    assert ck.d.eof
    assert ck.n == total and ck.crc == crc
    assert int.from_bytes(ck.tail[4:], "little") == total % (1 << 32)
    assert int.from_bytes(ck.tail[:4], "little") == crc
    print("gzip stream of %d bytes -> %d bytes in %.1f s (%.2f GB/s including the host side)" % (total, ck.comp, secs,
                                                                                                total / secs / 1e9))
