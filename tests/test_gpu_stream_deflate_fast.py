"""GPU tier: open runs of levels 0-4 (B200Z_END_NONE), by hand through the plan calls and inside the Deflater handle.
Tests named *small* also run on the CUDA emulator (tests/test_stream_deflate_fast.py)."""
import random
import resource
import time
import zlib

import numpy as np
import pytest

from fast_chain import chained, live_log, live_state, new_state, shift_position
from sharpziplib_b200 import _lib
from stream_chain import zlib_frame

pytestmark = pytest.mark.gpu


def plan_runner(z, level, strategy):
    """one run as a single-stream device plan: the engine state handed in and read back, the cut and its call reported"""
    import torch

    def run(hist, seg, pos_base, bit_base, calls, end_mode, state, cont):
        if level == 0:
            st = np.frombuffer(state, np.uint8).copy()
        else:
            st = [torch.from_numpy(np.frombuffer(state, np.uint8).copy()).cuda()]
        kw = dict(history=([len(hist)], [pos_base], [bit_base])) if cont else (dict(dict_lens=[len(hist)]) if hist else {})
        p = z.DeflatePlan([len(seg)], level=level, strategy=strategy, end_mode=end_mode, chunk_lens=[calls], state=st, **kw)
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
            cov, calls_at = p.cut()
            cut = (int(cov[0]), int(calls_at[0]))
        p.close()
        return out, nb, cut, (st.tobytes() if level == 0 else st[0].cpu().numpy().tobytes())
    return run


def model_runner(level, strategy):
    from test_stream_deflate_fast import model_lib, model_runner as mr
    return mr(model_lib(), level, strategy)


# ---- small: also on the emulator -----------------------------------------------------------------------------------
def small_data():
    from sharpziplib_b200 import datagen
    rng = np.random.default_rng(12)
    return (rng.integers(0, 256, 70000, dtype=np.uint8).tobytes() + datagen.silesia_mix(0, 60000, config=9).tobytes()
            + rng.integers(0, 256, 50000, dtype=np.uint8).tobytes())


def small_calls(n):
    rnd = random.Random(n)
    out, left = [], n
    while left:
        c = min(left, rnd.choice([1, 261, 262, 32768, 65273, 65274, 65275, rnd.randrange(1, 40000)]))
        out.append(c)
        left -= c
    return out


@pytest.mark.parametrize("level", [0, 1, 4])
def test_small_open_runs_match_oracle_and_model(z, oracle, level):
    from test_stream_deflate_fast import want_bytes
    data = small_data()
    calls = small_calls(len(data))
    for close in (0, 1):
        ch = chained(plan_runner(z, level, 0), level, data, calls, [40000, 50000], close)
        assert bytes(ch.out) == want_bytes(level, 0, data, calls, close)
        assert any(c > 0 for (_, _, _, c, _, _) in ch.log[:-1])
        m = chained(model_runner(level, 0), level, data, calls, [40000, 50000], close)
        assert live_log(level, ch.log) == live_log(level, m.log)


def test_small_open_runs_need_the_engine_state(z):
    import torch
    n = 100000
    with pytest.raises(z.B200zUnsupported):  # a schedule, but nowhere to write the cut
        z.DeflatePlan([n], level=1, end_mode=_lib.END_NONE, chunk_lens=[[n]])
    p = z.DeflatePlan([n], level=1, end_mode=_lib.END_NONE, chunk_lens=[[n]],
                      state=[torch.zeros(_lib.lib().b200z_engine_state_bytes(), dtype=torch.uint8, device="cuda")])
    with pytest.raises(z.InvalidOperationException):  # no run yet
        p.cut()
    p.close()
    p = z.DeflatePlan([n], level=0, end_mode=_lib.END_NONE, chunk_lens=[[n]], state=np.zeros(16, np.uint8))
    p.close()
    p = z.DeflatePlan([1000], level=6)
    arr = np.zeros(1, np.int32)
    assert _lib.lib().b200z_deflate_plan_get_cut_call(p._h, arr.ctypes.data, None) == _lib.E_STATE
    p.close()


# ---- plan level ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [0, 1, 4])
def test_open_runs_chained_by_hand(z, oracle, level):
    """every strategy and close against the oracle; run by run (covered, bits, call of the cut, engine state: live_state)
    the CPU model's"""
    from test_stream_deflate_fast import chains_for, want_bytes
    data, chains = chains_for(level)
    for strategy, close, calls, runs, m in chains:
        if level == 0 and strategy:
            continue
        ch = chained(plan_runner(z, level, strategy), level, data, calls, runs, close)
        assert bytes(ch.out) == want_bytes(level, strategy, data, calls, close), (strategy, close)
        assert live_log(level, ch.log) == live_log(level, m.log), (strategy, close)
        if close == 0:
            assert zlib_frame(level, ch.out, ch.adler) == want_bytes(level, strategy, data, calls, 0, nowrap=False)


@pytest.mark.parametrize("level", [0, 1, 4])
def test_position_beyond_4gib_is_the_same_phase(z, level):
    """a run whose engine stands k * 32768 bytes further on, past 2^32, writes the same bytes and leaves the same state
    as the CPU model"""
    from test_stream_deflate_fast import corpus, schedule
    data = corpus(4, 9)
    run = plan_runner(z, level, 0)
    calls = schedule(random.Random(level), 1_200_000)
    hist, seg = data[:32768 * 3], data[32768 * 3:32768 * 3 + 1_200_000]
    _, _, _, st = run(b"", hist, 0, 0, [len(hist)], _lib.END_FLUSH, new_state(level), False)
    P = len(hist)
    k = (2 ** 32 - P) // 32768 + 1
    for end_mode in (_lib.END_NONE, _lib.END_FINISH):
        a = run(hist[-32768:], seg, P, 3, calls, end_mode, st, True)
        b = run(hist[-32768:], seg, P + k * 32768, 3, calls, end_mode, shift_position(level, st, k), True)
        assert a == b, end_mode
        m = model_runner(level, 0)(hist[-32768:], seg, P, 3, calls, end_mode, st, True)
        assert a[1] == m[1] and a[0] == m[0][:len(a[0])] and live_state(level, a[3]) == live_state(level, m[3])
        assert a[2] == (m[2] if end_mode == _lib.END_NONE else None)


# ---- the Deflater handle -------------------------------------------------------------------------------------------
class _Sink:
    def __init__(self):
        self.buf = bytearray()

    def write(self, b):
        self.buf += b


@pytest.mark.parametrize("level", [0, 1])
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
    pos, calls = 0, [[], []]
    out_before = 0
    while pos < len(mixed):
        step = min(rnd.choice([1, 4097, 65536, 1 << 20, 3 << 20, 7 << 20]), (half if pos < half else len(mixed)) - pos)
        s.Write(mixed[pos:pos + step])
        calls[pos >= half].append(step)
        pos += step
        if pos == half:
            out_before = s.deflater_.TotalOut
            s.Flush()
    total_out_before = s.deflater_.TotalOut
    s.Finish()
    assert out_before > 0 and total_out_before > out_before
    want = oracle_calls(level, [(mixed[:half], calls[0]), (mixed[half:], calls[1])], nowrap=False)
    assert bytes(sink.buf) == want
    assert s.deflater_.TotalIn == len(mixed)
    assert s.deflater_.Adler == zlib.adler32(mixed)


def test_gzip_stream_over_4gib_level_0(z):
    """about 4.5 GiB through GZipOutputStream at level 0 in 1 MiB writes: inflates back (CRC-32 and length of the output
    equal the input's), ISIZE = TotalIn mod 2^32, and the host does not hold the input: peak RSS grows by far less"""
    from sharpziplib_b200 import datagen
    pool = datagen.log_stream(64 << 20).tobytes()
    total = (9 << 29) + 12345

    class Check:
        def __init__(self):
            self.d = zlib.decompressobj(31)
            self.crc = 0
            self.n = 0
            self.tail = b""

        def write(self, b):
            out = self.d.decompress(b)
            self.crc = zlib.crc32(out, self.crc)
            self.n += len(out)
            self.tail = (self.tail + bytes(b))[-8:]

    ck = Check()
    g = z.GZipOutputStream(ck, level=0)
    g.ModifiedTime = 0
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss << 10
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
    grew = (resource.getrusage(resource.RUSAGE_SELF).ru_maxrss << 10) - rss0
    ck.d.flush()
    assert ck.d.eof
    assert ck.n == total and ck.crc == crc
    assert int.from_bytes(ck.tail[4:], "little") == total % (1 << 32)
    assert int.from_bytes(ck.tail[:4], "little") == crc
    assert grew < total // 4, grew
    print("level 0 gzip stream of %d bytes in %.1f s, peak RSS grew by %.2f GiB" % (total, secs, grew / 2 ** 30))
