"""CPU tier: open runs of levels 5-9 (B200Z_END_NONE) on the CPU model.  Chained by hand through their cuts and entry
states and closed by a Finish / Flush-then-Finish / Flush run, they must give the oracle's bytes for the whole input."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from stream_chain import CLEAN, chained, random_runs, zlib_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model_lib():
    so = os.path.join(ROOT, "tests", "cpu_model", "_build", "libstream_model.so")
    srcs = [os.path.join(ROOT, "tests", "cpu_model", f) for f in ("stream_model.cpp", "model.cpp")]
    hdr = os.path.join(ROOT, "sharpziplib_b200", "csrc", "b200z_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs + [hdr]):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", os.path.dirname(hdr), "-o", so, srcs[0]])
    M = C.CDLL(so)
    M.model_deflate_open.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p]
    return M


def model_runner(M, level, strategy):
    def run(hist, mask, seg, pos_base, bit_base, end_mode, entry):
        buf = np.frombuffer(hist + bytes(seg) + b"\0", np.uint8).copy()
        hm = np.frombuffer(mask + b"\0", np.uint8).copy()
        cap = len(seg) + len(seg) // 8 + 1024
        out = np.zeros(cap, np.uint8)
        bits = C.c_uint64(0)
        ent = np.array(entry, np.int64)
        cut = np.zeros(4, np.int64)
        rc = M.model_deflate_open(buf.ctypes.data, len(hist) + len(seg), len(hist), pos_base, bit_base, hm.ctypes.data, level,
                                  strategy, end_mode, ent.ctypes.data, out.ctypes.data, cap, C.byref(bits), cut.ctypes.data)
        assert rc == 0, rc
        return out.tobytes(), bits.value, (int(cut[0]), tuple(int(x) for x in cut[1:]))
    return run


@pytest.fixture(scope="module")
def M():
    return model_lib()


def stream_corpus():
    """A log-like text stream with stretches of random bytes (stored blocks) and long repeats (matches pending at cuts)."""
    from sharpziplib_b200 import datagen
    rng = np.random.default_rng(2024)
    parts = []
    for k in range(22):
        parts.append(datagen.silesia_mix(k % 8, 700000 + 37 * k, config=8).tobytes())
        if k % 6 == 1:
            parts.append(rng.integers(0, 256, 1500000 + k, dtype=np.uint8).tobytes())
    return b"".join(parts)


def oracle_raw(oracle, data, level, strategy, pattern):
    return oracle.deflate(data, level=level, strategy=strategy, pattern=pattern)


def stats_of(chains, data):
    """what the cuts of the chains covered: pending matches, stored blocks behind a cut, cuts near slide positions"""
    pend_match = near_slide = 0
    for ch in chains:
        pos = 0
        for (_, _, covered, nxt) in ch.log[:-1]:
            pos += covered
            pend_match += nxt[0] == 1 and nxt[1] >= 3
            q = ch.dict_len + pos
            if q >= 65273 and min((q - 65273) % 32768, 32768 - (q - 65273) % 32768) < 300:
                near_slide += 1
    return pend_match, near_slide


def stored_after_cut(raw_cuts_bits, out):
    """block type of the first block behind each cut, read from the bit position where the cut left the stream"""
    types = []
    for b in raw_cuts_bits:
        byte, sh = divmod(b, 8)
        v = int.from_bytes(bytes(out[byte:byte + 2]) + b"\0\0", "little") >> sh
        types.append((v >> 1) & 3)
    return types


@pytest.mark.parametrize("level", [5, 6, 7, 8, 9])
def test_open_runs_match_oracle(M, oracle, level):
    data = stream_corpus()
    rnd = random.Random(level)
    chains = []
    stored_behind_cut = 0
    for strategy in (0, 1, 2):
        # every (strategy, close) pair comes up at some level
        close = (strategy + level) % 3
        want = {p: oracle_raw(oracle, data, level, strategy, p) for p in ((0,) if close == 0 else (1,))}
        if True:
            runs = random_runs(rnd, len(data), 4_000_000, 5_000_000)
            assert len(runs) >= 2
            ch = chained(model_runner(M, level, strategy), data, runs, close)
            ch.dict_len = 0
            assert bytes(ch.out) == want[0 if close == 0 else 1], (strategy, close, runs)
            chains.append(ch)
            stored_behind_cut += sum(t == 0 for t in stored_after_cut(ch.end_bits[:-1], ch.out))
        # zlib: the Adler-32 of the chain takes every covered byte once
        if close == 0:
            zl = oracle.deflate(data, level=level, nowrap=False, strategy=strategy)
            assert zlib_frame(level, ch.out, ch.adler) == zl
    assert stored_behind_cut > 0, "no stored block right behind a cut"


@pytest.mark.parametrize("level", [6, 9])
def test_cuts_with_pending_matches(M, oracle, level):
    """short open runs over text, so that many cuts happen: some leave a byte pending with a match of length >= 3 found at
    it (trap T10), which the next run has to take over"""
    data = stream_corpus()[:6_000_000]
    runs = random_runs(random.Random(level), len(data), 250_000, 350_000)
    ch = chained(model_runner(M, level, 0), data, runs, 0)
    ch.dict_len = 0
    assert bytes(ch.out) == oracle.deflate(data, level=level)
    pend_match, _ = stats_of([ch], data)
    assert pend_match > 0, "no cut with a pending match of length >= 3"


def test_open_runs_cut_near_slide_positions(M, oracle):
    """a cut within 300 bytes of a slide position (trap T8).  A preset dictionary in front moves the stream offset of the
    cut: its length is chosen so that the cut lands 100 bytes in front of a slide position."""
    from helpers import oracle_calls
    rng = np.random.default_rng(7)
    data = rng.integers(0, 256, 3_000_000, dtype=np.uint8).tobytes() + b"abcabcabd" * 200000
    text = stream_corpus()[:40000]
    run = model_runner(M, 6, 0)
    D = 20000
    for _ in range(4):
        ch = chained(run, data, [2_000_000], 0, dictionary=text[:D])
        r = (D + ch.log[0][2] - 65273) % 32768
        if min(r, 32768 - r) < 300:
            break
        D = (D - r - 100) % 32768 if r < 16384 else (D + 32768 - r - 100) % 32768
        D = max(D, 3)
    else:
        pytest.fail("no cut near a slide position")
    assert zlib_frame(6, ch.out, ch.adler, text[:D]) == oracle_calls(6, [(data, [len(data)])], dictionary=text[:D])


def test_open_runs_after_dictionary(M, oracle):
    from helpers import oracle_calls
    data = stream_corpus()[:13_000_000]
    dictionary = data[5_000_000:5_040_000]
    for level in (6, 9):
        ch = chained(model_runner(M, level, 0), data, [4_200_000, 4_700_000], 0, dictionary=dictionary)
        want = oracle_calls(level, [(data, [len(data)])], dictionary=dictionary)
        assert zlib_frame(level, ch.out, ch.adler, dictionary) == want


def test_entry_state_is_used(M):
    """at cuts with a pending match, entering the next run without the match gives other bytes (not at every such cut: a
    longer match one byte on makes the pending one irrelevant).  A clean start at the pending byte mostly repeats the
    search the previous run made there, so it is no test of the entry state."""
    data = stream_corpus()[:3_000_000]
    run = model_runner(M, 6, 0)
    ch = chained(run, data, random_runs(random.Random(6), len(data), 250_000, 350_000), 0)
    pos, tried, differ = 0, 0, 0
    for (_, _, covered, nxt) in ch.log[:-1]:
        pos += covered
        if nxt[0] == 1 and nxt[1] >= 3:
            hist, seg = data[pos - 32768:pos], data[pos:pos + 400_000]
            a = run(hist, bytes(32768), seg, pos, 0, 3, nxt)[:2]
            differ += a != run(hist, bytes(32768), seg, pos, 0, 3, (1, 2, 0))[:2]
            tried += 1
    assert tried > 0, "no cut with a pending match"
    assert differ > 0


def test_gpu_small_plan_tests_on_emulator():
    """the GPU tier's small plan tests, on the CUDA emulator (tests/cuda_emu)"""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"), "-q", "-x",
                        os.path.join(ROOT, "tests", "test_gpu_stream_deflate.py"), "-k", "small"],
                       capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
