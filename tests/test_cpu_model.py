"""CPU tier: the kernel decomposition (b200z_core.cuh, the same __host__ __device__ code the CUDA kernels call) executed
serially by tests/cpu_model/model.cpp must reproduce the oracle bit for bit."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

from helpers import corpus_small, oracle_calls as _oracle_calls, random_chunks as _random_chunks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def model():
    so = os.path.join(ROOT, "tests", "cpu_model", "_build", "libmodel.so")
    src = os.path.join(ROOT, "tests", "cpu_model", "model.cpp")
    hdr = os.path.join(ROOT, "sharpziplib_b200", "csrc", "b200z_core.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", os.path.dirname(hdr), "-o", so, src])
    M = C.CDLL(so)
    M.model_deflate.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]

    def run(d, level=6, strategy=0, flush_then_finish=0):
        a = np.frombuffer(d, dtype=np.uint8) if len(d) else np.zeros(1, np.uint8)
        cap = len(d) + len(d) // 8 + 1024
        out = np.zeros(cap, np.uint8)
        ol = C.c_uint64(0)
        rc = M.model_deflate(a.ctypes.data, len(d), level, strategy, flush_then_finish, out.ctypes.data, cap, C.byref(ol))
        assert rc == 0, rc
        return out[:ol.value].tobytes()
    return run


def test_model_matches_oracle(model, oracle):
    for name, d in corpus_small():
        for level in (5, 6, 9):
            assert model(d, level) == oracle.deflate(d, level=level), (name, level)
        assert model(d, 6, 0, 1) == oracle.deflate(d, level=6, pattern=1), name


def test_model_strategies(model, oracle):
    for name, d in corpus_small():
        if len(d) not in (1000, 70000):
            continue
        for strategy in (1, 2):
            assert model(d, 6, strategy) == oracle.deflate(d, level=6, strategy=strategy), (name, strategy)


def test_model_multi_slide(model, oracle):
    from sharpziplib_b200 import datagen
    for cls in (0, 4, 6):
        d = datagen.silesia_mix(cls, 400000, config=8).tobytes()
        assert model(d, 6) == oracle.deflate(d, level=6), cls


def test_model_fast_and_stored_levels(model, oracle):
    """levels 1-4 (serial DeflateFast engine, what k_fast runs) and level 0 (stored_run bookkeeping)"""
    from sharpziplib_b200 import datagen
    items = [(n, d) for n, d in corpus_small() if len(d) in (0, 3, 100, 4096, 70000)]
    items.append(("mix3_400k", datagen.silesia_mix(3, 400000, config=8).tobytes()))
    items.append(("zeros_300k", bytes(300000)))
    for name, d in items:
        for level in (0, 1, 2, 3, 4):
            assert model(d, level) == oracle.deflate(d, level=level), (name, level)
            assert model(d, level, 0, 1) == oracle.deflate(d, level=level, pattern=1), (name, level)


# ---- streams with history: preset dictionary, input after Flush() -------------------------------------------
class _SegmentedModel:
    """The bookkeeping of the Deflater handle in b200z_handles.cu (carried window image, uninserted-position mask, window
    phase, sub-byte tail), driving the CPU model segment by segment."""

    def __init__(self, root, level, strategy=0):
        so = os.path.join(root, "tests", "cpu_model", "_build", "libmodel.so")
        self.M = C.CDLL(so)
        self.M.model_deflate_ex.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int,
                                            C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        self.M.model_deflate_ex2.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int,
                                             C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                             C.c_uint64, C.POINTER(C.c_uint64)]
        # levels 0-4: what the engine carries between segments (head[] / prev[] / scalars), as k_fast keeps it in
        # b200z_history.engine_state
        self.state = np.zeros(self.M.model_state_bytes(), np.uint8)
        self.started = False
        self.level, self.strategy = level, strategy
        self.hist = bytearray()
        self.mask = bytearray()
        self.seen = 0
        self.tail_bits, self.tail_count = 0, 0
        self.out = bytearray()

    def remember(self, seg, uninserted=2):
        self.hist += seg
        m = bytearray(len(seg))
        for k in range(min(uninserted, len(seg))):
            m[len(seg) - 1 - k] = 1
        self.mask += m
        if len(self.hist) > 32768:
            cut = len(self.hist) - 32768
            del self.hist[:cut]
            del self.mask[:cut]
        self.seen += len(seg)

    def set_dictionary(self, d):
        if len(d) < 3:
            return
        self.remember(d[-32506:])

    def segment(self, seg, end_mode, chunks=None, busy_last=True):
        """chunks: the sizes of the SetInput calls that delivered `seg` (None: one call); busy_last: Deflate() was called
        behind the last of them before Flush() / Finish()"""
        H = len(self.hist)
        buf = np.frombuffer(bytes(self.hist) + bytes(seg) + b"\0", dtype=np.uint8).copy()
        mask = np.frombuffer(bytes(self.mask) + b"\0", dtype=np.uint8).copy()
        cap = len(seg) + len(seg) // 8 + 1024 + 5 * (len(chunks) if chunks else 0)
        out = np.zeros(cap, np.uint8)
        bits = C.c_uint64(0)
        if self.level >= 5 and chunks is None:
            rc = self.M.model_deflate_ex(buf.ctypes.data, H + len(seg), H, self.seen, self.tail_count, mask.ctypes.data,
                                         self.level, self.strategy, end_mode, out.ctypes.data, cap, C.byref(bits))
        else:
            if chunks:
                assert sum(chunks) == len(seg)
            cum = np.cumsum(np.array(chunks if chunks else [len(seg)], dtype=np.uint32), dtype=np.uint32)
            rc = self.M.model_deflate_ex2(buf.ctypes.data, H + len(seg), H, self.seen, self.tail_count, mask.ctypes.data,
                                          self.level, self.strategy, end_mode, cum.ctypes.data, len(cum), 1 if busy_last else 0,
                                          self.state.ctypes.data, 1 if self.started else 0, out.ctypes.data, cap,
                                          C.byref(bits))
        self.started = True
        assert rc == 0, rc
        nb = bits.value
        o = bytearray(out[:(nb + 7) // 8].tobytes())
        if o:
            o[0] |= self.tail_bits
        whole = nb // 8
        self.out += o[:whole]
        self.tail_count = nb & 7
        self.tail_bits = (o[whole] & ((1 << self.tail_count) - 1)) if self.tail_count else 0
        if end_mode == 0 and self.tail_count:
            self.out.append(self.tail_bits)
            self.tail_bits = self.tail_count = 0
        self.remember(seg)


def _oracle_segments(oracle_mod, level, segs, dictionary=None, strategy=0):
    """reference call sequence: [SetDictionary] (SetInput, Flush, drain)* SetInput, Finish, drain -- zlib framing stripped"""
    from oracle_lib import Deflater
    d = Deflater(level, nowrap=dictionary is None)
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
    for i, s in enumerate(segs):
        d.set_input(s)
        if i + 1 < len(segs):
            d.flush()
        else:
            d.finish()
        drain()
    return bytes(out)


def _model_segments(level, segs, dictionary=None, strategy=0):
    m = _SegmentedModel(ROOT, level, strategy)
    if dictionary is not None:
        m.set_dictionary(dictionary)
    for i, s in enumerate(segs):
        m.segment(s, 2 if i + 1 < len(segs) else 0)
    return bytes(m.out)


def test_model_dictionary(model, oracle):
    from sharpziplib_b200 import datagen
    text = datagen.gen_text(120000, 5).tobytes()
    for level in (1, 4, 5, 6, 9):
        for dlen in (2, 3, 100, 32506, 40000):
            dic = text[:dlen]
            data = text[20000:20000 + 70000]
            ref = _oracle_segments(oracle, level, [data], dictionary=dic)
            # zlib framing: 2 header bytes + 4 DICTID bytes in front, 4 Adler bytes behind
            assert ref[1] & 0x20
            got = _model_segments(level, [data], dictionary=dic)
            assert got == ref[6:-4], (level, dlen)


def test_model_flush_continue(model, oracle):
    from sharpziplib_b200 import datagen
    text = datagen.gen_text(300000, 9).tobytes()
    mixed = datagen.silesia_mix(4, 200000, config=3).tobytes()
    cases = [
        [text[:1000], text[1000:5000], text[5000:5001], text[5001:5003], text[5003:90000]],
        [text[:40000], text[40000:140000], text[140000:300000]],   # crosses the first window slides
        [mixed[:65000], mixed[65000:65300], mixed[65300:131000], b"", mixed[131000:]],
        [b"", text[:10], b"", text[10:20000]],
    ]
    for level in (5, 6, 9):
        for ci, segs in enumerate(cases):
            assert _model_segments(level, segs) == _oracle_segments(oracle, level, segs), (level, ci)


def test_model_random_segments_and_dictionaries(model, oracle):
    """seeded random call sequences: [SetDictionary] (SetInput, Flush)* SetInput, Finish with cuts at and around the window
    slide positions, levels 5-9, all strategies -- the segment bookkeeping of the Deflater handle over the kernel model"""
    import random
    from sharpziplib_b200 import datagen
    rnd = random.Random(77)
    special = [32768, 65272, 65273, 65274, 98041, 98042]
    for trial in range(14):
        n = rnd.choice([3000, 70000, 140000])
        d = datagen.silesia_mix(rnd.randrange(8), n, config=rnd.randrange(1, 9)).tobytes()
        cuts = sorted(min(len(d), rnd.choice([rnd.randrange(0, len(d) + 1)] + special)) for _ in range(rnd.randrange(1, 6)))
        segs = [d[a:b] for a, b in zip([0] + cuts, cuts + [len(d)])]
        level, strat = rnd.choice([5, 6, 7, 8, 9]), rnd.choice([0, 0, 0, 1, 2])
        dic = d[:rnd.choice([5, 1000, 32506, 50000])] if rnd.random() < 0.4 else None
        ref = _oracle_segments(oracle, level, segs, dictionary=dic, strategy=strat)
        if dic is not None:
            ref = ref[6:-4]
        assert _model_segments(level, segs, dictionary=dic, strategy=strat) == ref, (trial, n, cuts, level, strat)


# ---- levels 0-4: SetInput schedules (trap T9) and input after Flush() ----------------------------------------------
def _model_calls(level, segs, dictionary=None, busy_last=True):
    m = _SegmentedModel(ROOT, level)
    if dictionary is not None:
        m.set_dictionary(dictionary)
    for i, (seg, chunks) in enumerate(segs):
        m.segment(seg, 2 if i + 1 < len(segs) else 0, chunks=chunks, busy_last=busy_last)
    return bytes(m.out)


@pytest.mark.parametrize("level", [0, 1, 2, 3, 4])
def test_model_setinput_schedules_and_flush_levels_0_to_4(model, oracle, level):
    """DeflateStored / DeflateFast depend on how the input arrives (trap T9) and keep window-relative state across
    Flush(): the engine code the kernels run (stored_run / fe_run with a schedule, FastCarry / StoredCarry between
    segments) must reproduce the reference for arbitrary call sequences."""
    import random
    from sharpziplib_b200 import datagen
    rnd = random.Random(1000 + level)
    text = datagen.gen_text(400000, 31).tobytes()
    mixed = datagen.silesia_mix(3, 300000, config=5).tobytes()
    for trial in range(int(os.environ.get('B200Z_SCHED_TRIALS', '10'))):
        src = text if trial % 2 == 0 else mixed
        n = rnd.choice([0, 5, 3000, 66000, 140000, 250000])
        nseg = rnd.choice([1, 1, 2, 3, 5])
        cuts = sorted(rnd.randrange(0, n + 1) for _ in range(nseg - 1))
        bounds = [0] + cuts + [n]
        segs = []
        for a, b in zip(bounds[:-1], bounds[1:]):
            seg = src[a:b]
            chunks = _random_chunks(rnd, len(seg))
            segs.append((seg, chunks))
        busy_last = rnd.random() < 0.7
        dictionary = None
        if level != 0 and rnd.random() < 0.3:
            dictionary = src[-rnd.choice([3, 500, 32506, 40000]):]
        ref = _oracle_calls(level, segs, dictionary, busy_last)
        if dictionary is not None:
            ref = ref[6:-4]
        got = _model_calls(level, segs, dictionary, busy_last)
        assert got == ref, (level, trial, n, [len(s) for s, _ in segs], [c[:6] for _, c in segs], busy_last,
                            None if dictionary is None else len(dictionary))
        do = zlib.decompressobj(-15) if dictionary is None else zlib.decompressobj(-15, zdict=dictionary)
        back, whole = do.decompress(got), b"".join(s for s, _ in segs)
        # Finish() right behind an undrained SetInput at level 0 ends the stream early in the reference itself
        # (DeflateStored takes lastBlock = finish even while input is still outside the window, DeflaterEngine.cs:631):
        # reproduced, not repaired
        assert back == whole or (level == 0 and not busy_last and whole.startswith(back))
