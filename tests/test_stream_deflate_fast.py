"""CPU tier: open runs of levels 0-4 (B200Z_END_NONE) on the CPU model.  Chained by hand through their cuts, with the
engine state and the rest of the cut's SetInput call carried over, and closed by a Finish / Flush-then-Finish / Flush run,
they must give the oracle's bytes for the same SetInput schedule."""
import ctypes as C
import functools
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from fast_chain import chained, new_state, shift_position
from helpers import oracle_calls
from stream_chain import zlib_frame
from test_stream_deflate import stored_after_cut

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model_lib():
    so = os.path.join(ROOT, "tests", "cpu_model", "_build", "libfast_stream_model.so")
    srcs = [os.path.join(ROOT, "tests", "cpu_model", f) for f in ("fast_stream_model.cpp", "model.cpp")]
    hdr = os.path.join(ROOT, "sharpziplib_b200", "csrc", "b200z_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + [hdr]):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", os.path.dirname(hdr), "-o", so, srcs[0]])
    M = C.CDLL(so)
    M.model_deflate_fast_run.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                                         C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64,
                                         C.POINTER(C.c_uint64), C.c_void_p]
    return M


def model_runner(M, level, strategy):
    def run(hist, seg, pos_base, bit_base, calls, end_mode, state, cont):
        buf = np.frombuffer(hist + seg + b"\0", np.uint8).copy()
        cum = np.cumsum(np.array(calls, np.int64)).astype(np.uint32) if calls else np.zeros(1, np.uint32)
        st = np.frombuffer(state, np.uint8).copy()
        cap = len(seg) + len(seg) // 8 + 1024
        out = np.zeros(cap, np.uint8)
        bits = C.c_uint64(0)
        cut = np.zeros(2, np.int64)
        rc = M.model_deflate_fast_run(buf.ctypes.data, len(hist) + len(seg), len(hist), pos_base & 0xFFFFFFFF, bit_base, level,
                                      strategy, end_mode, cum.ctypes.data, len(calls), 1, st.ctypes.data, int(cont),
                                      out.ctypes.data, cap, C.byref(bits), cut.ctypes.data)
        assert rc == 0, rc
        return out.tobytes(), bits.value, (int(cut[0]), int(cut[1])), st.tobytes()
    return run


@pytest.fixture(scope="module")
def M():
    return model_lib()


def corpus(n_parts=10, seed=2025):
    """text with stretches of random bytes (stored blocks, level 0's MAX_DIST cuts) and long repeats (long matches)"""
    from sharpziplib_b200 import datagen
    rng = np.random.default_rng(seed)
    parts = []
    for k in range(n_parts):
        parts.append(datagen.silesia_mix(k % 8, 400000 + 37 * k, config=8).tobytes())
        if k % 3 == 1:
            parts.append(rng.integers(0, 256, 300000 + k, dtype=np.uint8).tobytes())
        if k % 4 == 2:
            parts.append(bytes(rng.integers(0, 256, 97, dtype=np.uint8)) * 3000)
    return b"".join(parts)


def schedule(rnd, n):
    """SetInput sizes as DeflaterOutputStream users make them: stretches of one style each -- 1-byte calls, the window
    edges (261, 262, 32768, 65273-65275), sizes anywhere below 70000, and large writes"""
    out, left = [], n
    while left:
        style = rnd.choice(["tiny", "edges", "mixed", "large"])
        for _ in range(rnd.randrange(1, 40)):
            if style == "tiny":
                c = rnd.choice([1, 1, 1, 2, 3])
            elif style == "edges":
                c = rnd.choice([1, 261, 262, 32768, 65273, 65274, 65275])
            elif style == "mixed":
                c = rnd.randrange(1, 70000)
            else:
                c = rnd.randrange(200000, 1500000)
            c = min(c, left)
            out.append(c)
            left -= c
            if not left:
                break
    return out


def run_lens(rnd, n, lo, hi):
    out, left = [], n
    while left > 2 * hi:
        L = rnd.randrange(lo, hi)
        out.append(L)
        left -= L
    return out


def want_bytes(level, strategy, data, calls, close, dictionary=None, nowrap=True):
    segs = [(data, calls)] if close == 0 else [(data, calls), (b"", [])]
    from oracle_lib import Deflater

    if strategy == 0:
        return oracle_calls(level, segs, dictionary=dictionary, nowrap=nowrap)
    # oracle_calls with a strategy: the same call sequence
    d = Deflater(level, nowrap=nowrap)
    d.set_strategy(strategy)
    if dictionary is not None:
        d.set_dictionary(dictionary)
    out = bytearray()

    def drain():
        while True:
            b = d.deflate(65536)
            if not b:
                break
            out.extend(b)
    for i, (seg, chunks) in enumerate(segs):
        pos = 0
        for c in chunks:
            d.set_input(seg[pos:pos + c])
            pos += c
            drain()
        (d.flush if i + 1 < len(segs) else d.finish)()
        drain()
    return bytes(out)


@functools.lru_cache(maxsize=None)
def chains_for(level):
    """the chains of one level: every strategy, every close; (strategy, close, calls, runs, chain) each"""
    M = model_lib()
    data = corpus()
    rnd = random.Random(40 + level)
    out = []
    for strategy in (0, 1, 2):
        for close in (0, 1, 2):
            calls = schedule(rnd, len(data))
            runs = run_lens(rnd, len(data), 300_000, 1_500_000)
            out.append((strategy, close, calls, runs, chained(model_runner(M, level, strategy), level, data, calls, runs, close)))
    return data, out


@pytest.mark.parametrize("level", [0, 1, 2, 3, 4])
def test_open_runs_match_oracle(oracle, level):
    data, chains = chains_for(level)
    for strategy, close, calls, runs, ch in chains:
        if level == 0 and strategy:
            continue  # (DeflateStored has no strategy)
        want = want_bytes(level, strategy, data, calls, close)
        assert bytes(ch.out) == want, (strategy, close)
        assert sum(c > 0 for (_, _, _, c, _, _) in ch.log[:-1]) >= 2
        if close == 0:
            assert zlib_frame(level, ch.out, ch.adler) == want_bytes(level, strategy, data, calls, 0, nowrap=False)


def _kinds(level):
    data, chains = chains_for(level)
    k = dict(partly=0, at_end=0, before=0, near_slide=0, stored_behind=0)
    for strategy, close, calls, runs, ch in chains:
        for (base, covered, (c0, c1), got) in ch.cuts:
            k["partly"] += got < c1
            k["at_end"] += got == c1
            k["before"] += covered < c0  # the block closed on bytes of an earlier call, after this call's Deflate() began
            pos = base + covered
            r = (pos - 65273) % 32768
            k["near_slide"] += pos >= 65273 and min(r, 32768 - r) < 300
        if level:
            k["stored_behind"] += sum(t == 0 for t in stored_after_cut(
                [b for b, (_, _, _, c, _, _) in zip(ch.end_bits[:-1], ch.log[:-1]) if c], ch.out))
    return k


def stored_block_lengths(out, end):
    """(length, last) of the stored blocks of a level 0 stream up to byte `end`"""
    pos, res = 0, []
    while pos + 5 <= end:
        n = out[pos + 1] | out[pos + 2] << 8
        res.append((n, out[pos] & 1))
        pos += 5 + n
    return res


def test_corpus_has_every_kind_of_cut():
    """the chains above cut where the call of the cut is partly in the window, where the window holds the whole call
    (inputOff at its end), where the block closed in front of the call's first byte (the next run's first call then
    begins inside an earlier call), within 300 bytes of a slide position; a stored block follows a cut; level 0 closes
    blocks by MAX_BLOCK_SIZE and by MAX_DIST"""
    total = dict(partly=0, at_end=0, before=0, near_slide=0, stored_behind=0)
    for level in (0, 1, 2, 3, 4):
        for key, v in _kinds(level).items():
            total[key] += v
    assert all(v > 0 for v in total.values()), total
    data, chains = chains_for(0)
    lens = []
    for _, _, _, _, ch in chains:
        lens += [n for n, last in stored_block_lengths(ch.out, ch.end_bits[-2] // 8) if not last]
    assert sum(n == 65531 for n in lens) > 0, "no block cut by MAX_BLOCK_SIZE"
    assert sum(32506 <= n < 65531 for n in lens) > 0, "no block cut by MAX_DIST"


@pytest.mark.parametrize("level", [1, 4])
def test_open_runs_after_dictionary(M, oracle, level):
    data = corpus(4, 7)
    dictionary = data[300_000:340_000]
    rnd = random.Random(level)
    calls = schedule(rnd, len(data))
    ch = chained(model_runner(M, level, 0), level, data, calls, run_lens(rnd, len(data), 200_000, 600_000), 0,
                 dictionary=dictionary)
    assert sum(c > 0 for (_, _, _, c, _, _) in ch.log[:-1]) >= 2
    want = want_bytes(level, 0, data, calls, 0, dictionary=dictionary, nowrap=False)
    assert zlib_frame(level, ch.out, ch.adler, dictionary) == want


@pytest.mark.parametrize("level", [0, 1, 4])
def test_position_beyond_4gib_is_the_same_phase(M, level):
    """a run whose engine stands k * 32768 bytes further on, past 2^32, writes the same bytes and leaves the same state"""
    data = corpus(4, 9)
    run = model_runner(M, level, 0)
    rnd = random.Random(level)
    calls = schedule(rnd, 1_200_000)
    hist, seg = data[:32768 * 3], data[32768 * 3:32768 * 3 + 1_200_000]
    # the state behind a first run over `hist` (several slides)
    _, _, _, st = run(b"", hist, 0, 0, [len(hist)], 2, new_state(level), False)
    P = len(hist)
    k = (2 ** 32 - P) // 32768 + 1
    for end_mode in (3, 0):
        a = run(hist[-32768:], seg, P, 3, calls, end_mode, st, True)
        b = run(hist[-32768:], seg, P + k * 32768, 3, calls, end_mode, shift_position(level, st, k), True)
        assert a == b, end_mode
        assert a[2][0] > 0 or end_mode != 3


def test_gpu_small_plan_tests_on_emulator():
    """the GPU tier's small plan tests of levels 0-4, on the CUDA emulator (tests/cuda_emu)"""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"), "-q", "-x",
                        os.path.join(ROOT, "tests", "test_gpu_stream_deflate_fast.py"), "-k", "small"],
                       capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
