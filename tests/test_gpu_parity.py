"""GPU tier (run with -m gpu on an H100): every CUDA path against the oracle, through the C-ABI."""
import io
import json
import os
import zlib

import numpy as np
import pytest

from helpers import corpus_small, crafted_t8, oracle_calls
from sharpziplib_b200 import datagen

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_fixtures.json")))


def test_native_library_is_loaded(z):
    z.deflate_batch([b"abcabcabc"], level=6)
    maps = open("/proc/self/maps").read()
    assert "libb200z.so" in maps


# ---- checksums -------------------------------------------------------------------------------------------
def test_checksum_kats(z):
    for k in GOLD["checksum_kats"]["crc32"]:
        c = z.Crc32()
        c.Update(k["ascii"].encode())
        assert c.Value == k["value"]
    a = z.Adler32()
    assert a.Value == 1
    a.Update(b"123456789")
    assert a.Value == 0x091E01DE
    a.Reset()
    assert a.Value == 1
    c = z.Crc32()
    c.Update(b"123456789" * 4, 6, 18)  # unaligned slice (ChecksumTests.cs:139-146)
    assert c.Value == 0x31CA9A2E


def test_checksum_sizes_and_running_updates(z, oracle):
    from sharpziplib_b200 import datagen
    for n in (1, 3, 127, 128, 129, 4095, 32767, 32768, 32769, 65537, 1000003, 5 << 20):
        d = datagen.Rng(n).bytes(n).tobytes()
        c = z.Crc32()
        c.Update(d)
        a = z.Adler32()
        a.Update(d)
        assert c.Value == oracle.crc32(d) == zlib.crc32(d), n
        assert a.Value == oracle.adler32(d) == zlib.adler32(d), n
        c2 = z.Crc32()
        a2 = z.Adler32()
        for lo, hi in ((0, n // 3), (n // 3, n // 3 + 1), (n // 3 + 1, n)):
            c2.Update(d[lo:hi])
            a2.Update(d[lo:hi])
        assert c2.Value == c.Value and a2.Value == a.Value
    c = z.Crc32()
    for b in b"123456789":
        c.Update(b)  # Update(int)
    assert c.Value == 0xCBF43926


def test_checksum_batch_device(z, oracle):
    import torch
    from sharpziplib_b200 import datagen
    bufs = [datagen.silesia_mix(i, 1000 + 37000 * i).tobytes() for i in range(9)]
    off = np.zeros(len(bufs), dtype=np.int64)
    lens = np.array([len(b) for b in bufs], dtype=np.int64)
    off[1:] = np.cumsum(lens + 3)[:-1]  # deliberately unaligned offsets
    blob = np.zeros(int(off[-1] + lens[-1]), dtype=np.uint8)
    for o, b in zip(off, bufs):
        blob[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    d = torch.from_numpy(blob).cuda()
    for kind, ref, init in ((0, oracle.crc32, 0), (1, oracle.adler32, 1)):
        val = torch.full((len(bufs),), init, dtype=torch.int64).to(torch.uint32).cuda() if hasattr(torch, "uint32") else None
        v = torch.from_numpy(np.full(len(bufs), init, dtype=np.uint32).view(np.int32)).cuda()
        rc = z.lib().b200z_checksum_batch_device(kind, d.data_ptr(), off.ctypes.data, lens.ctypes.data, len(bufs),
                                                v.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert rc == 0, z.lib().b200z_last_error()
        torch.cuda.synchronize()
        got = v.cpu().numpy().view(np.uint32)
        assert [int(x) for x in got] == [ref(b) for b in bufs]


# ---- deflate ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [0, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_deflate_parity_small_corpus(z, oracle, level):
    names, bufs = zip(*corpus_small())
    outs, _ = z.deflate_batch(list(bufs), level=level)
    for name, d, o in zip(names, bufs, outs):
        assert o == oracle.deflate(d, level=level), (name, level)


def test_deflate_default_level_is_6(z, oracle):
    d = corpus_small()[20][1]
    assert z.deflate_batch([d], level=-1)[0][0] == oracle.deflate(d, level=6)


@pytest.mark.parametrize("strategy", [1, 2])
def test_deflate_strategies(z, oracle, strategy):
    items = [(n, d) for n, d in corpus_small() if len(d) in (1000, 20000, 70000)]
    outs, _ = z.deflate_batch([d for _, d in items], level=6, strategy=strategy)
    for (name, d), o in zip(items, outs):
        assert o == oracle.deflate(d, level=6, strategy=strategy), (name, strategy)


def test_deflate_flush_then_finish_pattern(z, oracle):
    # Write(all) -> Flush() -> Finish(): the reference's own round-trip pattern (InflaterDeflaterTests.cs:49-62)
    items = [(n, d) for n, d in corpus_small() if len(d) in (0, 1, 100, 4096, 70000)]
    outs, _ = z.deflate_batch([d for _, d in items], level=6, end_mode=1)
    for (name, d), o in zip(items, outs):
        assert o == oracle.deflate(d, level=6, pattern=1), name
        assert zlib.decompress(o, -15) == d


def test_deflate_zlib_wrapper(z, oracle):
    items = [d for _, d in corpus_small() if len(d) in (0, 10, 4096, 70000)]
    for level in (5, 6, 7, 9):
        outs, checks = z.deflate_batch(items, level=level, wrap=1)
        for d, o, c in zip(items, outs, checks):
            assert o == oracle.deflate(d, level=level, nowrap=False), level
            assert int(c) == zlib.adler32(d)


def test_deflate_window_slides_and_t8(z, oracle):
    from sharpziplib_b200 import datagen
    bufs = [crafted_t8(), crafted_t8(40000)]
    bufs += [datagen.silesia_mix(c, 600000 + 12345 * c, config=7).tobytes() for c in (0, 3, 4, 6)]
    bufs += [bytes(200000), b"abcdefgh" * 40000]
    outs, _ = z.deflate_batch(bufs, level=6)
    for d, o in zip(bufs, outs):
        assert o == oracle.deflate(d, level=6)


def test_deflate_long_single_streams(z, oracle):
    """C4 shape in small: one long stream is parsed by hundreds of speculative chunks that are then stitched"""
    from sharpziplib_b200 import datagen
    bufs = [datagen.log_stream(16 << 20).tobytes(), datagen.gen_db(5 << 20, 77).tobytes(), bytes(3 << 20),
            datagen.Rng(9).bytes(2 << 20).tobytes()]
    outs, _ = z.deflate_batch(bufs, level=6)
    refs = oracle.batch(0, bufs, level=6, threads=4)
    assert outs == refs
    back, used, status = z.inflate_batch(outs, [len(b) for b in bufs])
    assert back == bufs


def test_deflate_c3_shape_parity_and_properties(z, oracle):
    """64 buffers of the C3 shape (256 KiB Silesia-mix): bit-exact vs the oracle, valid deflate, round trip."""
    from sharpziplib_b200 import datagen
    bufs = [datagen.silesia_mix(i, 262144).tobytes() for i in range(64)]
    outs, _ = z.deflate_batch(bufs, level=6)
    refs = oracle.batch(0, bufs, level=6, threads=8)
    assert outs == refs
    back, used, status = z.inflate_batch(outs, [len(b) for b in bufs])
    assert back == bufs and [int(u) for u in used] == [len(o) for o in outs]


@pytest.mark.parametrize("level", [0, 1, 4])
def test_deflate_fast_and_stored_levels(z, oracle, level):
    """DeflateFast (levels 1-4) and DeflateStored (0): window slides, flush pattern, zlib wrapper, strategies."""
    from sharpziplib_b200 import datagen
    bufs = [datagen.silesia_mix(c, 300000 + 7777 * c, config=6).tobytes() for c in range(8)] + [bytes(250000), crafted_t8()]
    outs, _ = z.deflate_batch(bufs, level=level)
    assert outs == [oracle.deflate(b, level=level) for b in bufs]
    outs, _ = z.deflate_batch(bufs[:4], level=level, end_mode=1)
    assert outs == [oracle.deflate(b, level=level, pattern=1) for b in bufs[:4]]
    outs, checks = z.deflate_batch(bufs[:4], level=level, wrap=1)
    assert outs == [oracle.deflate(b, level=level, nowrap=False) for b in bufs[:4]]
    if level:
        for strategy in (1, 2):
            outs, _ = z.deflate_batch(bufs[:3], level=level, strategy=strategy)
            assert outs == [oracle.deflate(b, level=level, strategy=strategy) for b in bufs[:3]]


@pytest.mark.parametrize("head", ["pool", "smem"])
@pytest.mark.parametrize("level", [1, 2, 3, 4])
def test_deflate_fast_group_steps_both_table_layouts(z, oracle, level, head, monkeypatch):
    """k_fast's warp-wide group steps (DeflaterEngine.cs:651-739 taken 32 loop tops at a time) with head[] in the global pool
    (many streams: several CTAs per SM) and in shared memory (few streams), and the same kernel with every loop top on lane 0:
    all three give the oracle's bytes.  Long repeats (covered lanes), incompressible bytes, runs of one byte (chains through
    the group itself), streams that end inside a group, a window slide."""
    from sharpziplib_b200 import datagen
    import numpy as np
    rng = np.random.default_rng(level)
    bufs = [datagen.silesia_mix(c, 90000 + 4099 * c, config=7).tobytes() for c in range(8)]
    bufs += [bytes(70000), b"ab" * 40000, rng.integers(0, 256, 50000, dtype=np.uint8).tobytes(), crafted_t8()]
    bufs += [datagen.text_buffer(1, k, config=7).tobytes() for k in (1, 2, 3, 261, 262, 263, 293, 294, 300, 555, 4096)]
    rep = rng.integers(0, 4, 3000, dtype=np.uint8).tobytes()
    bufs += [rep * 30, (rep[:700] + bytes(range(256))) * 120]
    refs = [oracle.deflate(b, level=level) for b in bufs]
    monkeypatch.setenv("B200Z_FAST_HEAD", head)
    outs, _ = z.deflate_batch(bufs, level=level)
    assert outs == refs
    if head == "pool":
        monkeypatch.setenv("B200Z_FAST_GROUP", "0")
        outs, _ = z.deflate_batch(bufs, level=level)
        assert outs == refs


def _drain(d):
    out = bytearray()
    buf = bytearray(65536)
    while True:
        k = d.Deflate(buf)
        if k <= 0:
            break
        out += buf[:k]
    return bytes(out)


def _ref_segments(level, segs, dictionary=None, nowrap=True, strategy=0):
    from oracle_lib import Deflater
    d = Deflater(level, nowrap=nowrap)
    d.set_strategy(strategy)
    if dictionary is not None:
        d.set_dictionary(dictionary)
    out = bytearray()
    for i, s in enumerate(segs):
        d.set_input(s)
        # (no Deflate() between SetInput and Flush()/Finish(): the handle sees that and runs the engines the same way --
        # at level 0 this order even makes the reference drop input behind a size-triggered block, DeflaterEngine.cs:629-641)
        d.flush() if i + 1 < len(segs) else d.finish()
        while True:
            b = d.deflate(65536)
            if not b:
                break
            out += b
    return bytes(out), d.adler & 0xFFFFFFFF, d.total_in, d.total_out


def _gpu_segments(z, level, segs, dictionary=None, nowrap=True, strategy=0):
    d = z.Deflater(level, nowrap)
    d.SetStrategy(strategy)
    if dictionary is not None:
        d.SetDictionary(dictionary)
    out = bytearray()
    for i, s in enumerate(segs):
        d.SetInput(s)
        d.Flush() if i + 1 < len(segs) else d.Finish()
        out += _drain(d)
    return bytes(out), d.Adler & 0xFFFFFFFF, d.TotalIn, d.TotalOut


@pytest.mark.parametrize("level", [5, 6, 9])
def test_deflater_input_after_flush(z, oracle, level):
    """SetInput after a sync Flush(): window, hash chains, slide phase and the sub-byte tail carry over (levels 5-9)"""
    text = datagen.gen_text(300000, 9).tobytes()
    mixed = datagen.silesia_mix(4, 200000, config=3).tobytes()
    cases = [
        [text[:1000], text[1000:5000], text[5000:5001], text[5001:5003], text[5003:90000]],
        [text[:40000], text[40000:140000], text[140000:300000]],
        [mixed[:65000], mixed[65000:65300], mixed[65300:131000], b"", mixed[131000:]],
        [b"", text[:10], b"", text[10:20000]],
        [crafted_t8()[:65273], crafted_t8()[65273:]],
    ]
    for ci, segs in enumerate(cases):
        for nowrap in (True, False):
            assert _gpu_segments(z, level, segs, nowrap=nowrap) == _ref_segments(level, segs, nowrap=nowrap), (ci, nowrap)
    assert _gpu_segments(z, level, cases[1], strategy=1) == _ref_segments(level, cases[1], strategy=1)


@pytest.mark.parametrize("level", [0, 1, 4, 5, 6, 9])
def test_deflater_preset_dictionary(z, oracle, level):
    """Deflater.SetDictionary: FDICT header + DICTID, dictionary tail as match history (all levels)"""
    text = datagen.gen_text(120000, 5).tobytes()
    data = text[20000:90000]
    for dlen in (2, 3, 100, 32506, 40000):
        dic = text[:dlen]
        got = _gpu_segments(z, level, [data], dictionary=dic, nowrap=False)
        assert got == _ref_segments(level, [data], dictionary=dic, nowrap=False), dlen
        assert got[0][1] & 0x20
    if level >= 5:  # dictionary, then input after a flush
        segs = [data[:30000], data[30000:30002], data[30002:]]
        assert _gpu_segments(z, level, segs, dictionary=text[:5000], nowrap=False) == \
            _ref_segments(level, segs, dictionary=text[:5000], nowrap=False)


def test_dictionary_state_errors(z):
    d = z.Deflater(6, True)
    with pytest.raises(Exception):  # a raw deflater never is in INIT_STATE (Deflater.cs:206, :561)
        d.SetDictionary(b"hello hello")
    d = z.Deflater(6, False)
    d.SetDictionary(b"hello hello")
    with pytest.raises(Exception):
        d.SetDictionary(b"twice")
    i = z.Inflater(False)
    with pytest.raises(Exception):  # "Dictionary is not needed"
        i.SetDictionary(b"abc")


def test_unsupported_sequences_fail_loudly(z, oracle):
    from oracle_lib import Deflater as RefDeflater
    d = z.Deflater(6, True)
    d.SetInput(b"abc" * 100)
    d.Flush()
    got = _drain(d)
    with pytest.raises(z.B200zUnsupported):
        d.SetLevel(1)  # DeflaterEngine.SetLevel in mid-stream flushes a block first (trap T17): not accelerated, not emulated
    d.SetStrategy(1)  # behind a completed Flush() the engine has nothing left: the switch is exact
    d.SetInput(b"xyz" * 100)
    with pytest.raises(z.B200zUnsupported):
        d.SetStrategy(2)  # ... but not while input is held: the reference would switch somewhere inside it
    d.Finish()
    got += _drain(d)
    r = RefDeflater(6, nowrap=True)
    want = bytearray()
    for seg, last in ((b"abc" * 100, False), (b"xyz" * 100, True)):
        r.set_input(seg)
        r.finish() if last else r.flush()
        while True:
            b = r.deflate(65536)
            if not b:
                break
            want += b
        if not last:
            r.set_strategy(1)
    assert got == bytes(want)


def test_inflater_preset_dictionary(z, oracle):
    from oracle_lib import Deflater
    text = datagen.gen_text(150000, 7).tobytes()
    for dlen, level in ((100, 6), (32506, 9), (50000, 1), (40000, 0)):
        dic, data = text[:dlen], text[60000:150000]
        comp = oracle_calls(level, [(data, [len(data)])], dic, True)  # SetInput, Deflate until it needs input, Finish
        adler = zlib.adler32(data)
        inf = z.Inflater(False)
        inf.SetInput(comp)
        buf = bytearray(len(data) + 100)
        assert inf.Inflate(buf) == 0 and inf.IsNeedingDictionary
        assert (inf.Adler & 0xFFFFFFFF) == int.from_bytes(comp[2:6], "big")
        with pytest.raises(z.SharpZipBaseException):  # "Wrong adler checksum"
            inf.SetDictionary(dic[:-1] + b"?")
        inf.SetDictionary(dic)
        got = bytearray()
        while not inf.IsFinished:
            k = inf.Inflate(buf)
            if k == 0 and inf.IsNeedingInput:
                break
            got += buf[:k]
        assert bytes(got) == data and inf.IsFinished, (dlen, level)
        assert (inf.Adler & 0xFFFFFFFF) == (adler & 0xFFFFFFFF)


def test_plan_run_in_two_stages(z, oracle):
    """b200z_plan_run_stages: SEARCH then ENCODE equals one run (levels 5-9 split, the others run whole in ENCODE)"""
    import torch
    bufs = [datagen.silesia_mix(c, 150000 + 999 * c, config=2).tobytes() for c in range(6)]
    for level in (6, 2, 0):
        plan = z.DeflatePlan([len(b) for b in bufs], level=level)
        blob = np.zeros(plan.in_bytes, np.uint8)
        for o, b in zip(plan.in_offsets, bufs):
            blob[o:o + len(b)] = np.frombuffer(b, np.uint8)
        d_in = torch.from_numpy(blob).cuda()
        d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(plan.n, dtype=torch.int64, device="cuda")
        d_st = torch.ones(plan.n, dtype=torch.int32, device="cuda")
        plan.run(d_in, d_out, d_len, d_st, stages=z.STAGE_SEARCH)
        plan.run(d_in, d_out, d_len, d_st, stages=z.STAGE_ENCODE)
        torch.cuda.synchronize()
        assert d_st.cpu().tolist() == [0] * plan.n
        for i, b in enumerate(bufs):
            o = int(plan.out_offsets[i])
            assert d_out[o:o + int(d_len[i])].cpu().numpy().tobytes() == oracle.deflate(b, level=level), (level, i)


def test_device_plans_with_dictionaries(z, oracle):
    """batch form: every stream of a plan with its own preset dictionary in front of its data"""
    import torch
    text = datagen.gen_text(200000, 11).tobytes()
    items = [(text[:1000], text[50000:120000]), (text[1000:33506], text[100000:200000]), (b"", text[:5000]), (text[:40], b"")]
    lens = [len(d) for _, d in items]
    dls = [len(k) for k, _ in items]
    for level in (1, 6):
        plan = z.DeflatePlan(lens, level=level, dict_lens=dls)
        blob = np.zeros(plan.in_bytes, np.uint8)
        for i, (k, d) in enumerate(items):
            o = int(plan.in_offsets[i])
            blob[o:o + len(k) + len(d)] = np.frombuffer(k + d, np.uint8)
            assert int(plan.data_offsets[i]) == o + len(k)
        d_in = torch.from_numpy(blob).cuda()
        d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(plan.n, dtype=torch.int64, device="cuda")
        d_st = torch.zeros(plan.n, dtype=torch.int32, device="cuda")
        plan.run(d_in, d_out, d_len, d_st)
        torch.cuda.synchronize()
        assert d_st.cpu().tolist() == [0] * plan.n
        outs = []
        for i, (k, d) in enumerate(items):
            o = int(plan.out_offsets[i])
            got = d_out[o:o + int(d_len[i])].cpu().numpy().tobytes()
            want = _ref_segments(level, [d], dictionary=k, nowrap=False)[0]
            want = want[6:-4]  # zlib framing: header + DICTID in front, Adler-32 behind
            assert got == want, (level, i)
            outs.append(got)
        # and back through an inflate plan with the same dictionaries
        ip = z.InflatePlan([len(o) for o in outs], [l + 64 for l in lens], dict_lens=dls)
        blob = np.zeros(ip.in_bytes, np.uint8)
        for i, (k, _) in enumerate(items):
            o = int(ip.in_offsets[i])
            blob[o:o + len(k) + len(outs[i])] = np.frombuffer(k + outs[i], np.uint8)
        d_in = torch.from_numpy(blob).cuda()
        d_out = torch.zeros(ip.out_bytes, dtype=torch.uint8, device="cuda")
        d_used = torch.zeros(ip.n, dtype=torch.int64, device="cuda")
        ip.run(d_in, d_out, d_len, d_st, None, d_used)
        torch.cuda.synchronize()
        assert d_st.cpu().tolist() == [0] * ip.n
        for i, (_, d) in enumerate(items):
            o = int(ip.out_offsets[i])
            assert d_out[o:o + int(d_len[i])].cpu().numpy().tobytes() == d, (level, i)


# ---- inflate ---------------------------------------------------------------------------------------------
def test_inflate_reference_fixtures(z):
    raw = bytes.fromhex(GOLD["inflate_ok"]["raw_hex"])
    out, used, st = z.inflate_batch([raw], [64])
    assert out[0] == b"testfile contents\n" and int(used[0]) == 20 and int(st[0]) == 0
    bad = bytes.fromhex(GOLD["inflate_zero_codelength"]["raw_hex"])
    out, used, st = z.inflate_batch([bad], [1 << 16], raise_on_error=False)
    assert int(st[0]) & 0xFF == 3 and (int(st[0]) >> 8) == 5  # E_DATA / "Encountered invalid codelength 0"
    with pytest.raises(z.SharpZipBaseException):
        z.inflate_batch([bad], [1 << 16])


def test_inflate_all_oracle_levels_and_zlib_streams(z, oracle):
    items = [d for _, d in corpus_small() if len(d) >= 100]
    for level in range(10):
        comp = [oracle.deflate(d, level=level) for d in items]  # stored (0), fast (1-4), lazy (5-9) producers
        out, used, st = z.inflate_batch(comp, [len(d) for d in items])
        assert out == items and [int(u) for u in used] == [len(c) for c in comp]
    for level in (1, 6, 9):
        comp = []
        for d in items:
            co = zlib.compressobj(level, zlib.DEFLATED, -15)
            comp.append(co.compress(d) + co.flush())
        out, used, st = z.inflate_batch(comp, [len(d) for d in items])
        assert out == items
    # sync-flush streams: empty static blocks in the middle (trap T6)
    comp = [oracle.deflate(d, level=6, pattern=1) for d in items]
    out, _, _ = z.inflate_batch(comp, [len(d) for d in items])
    assert out == items


def test_inflate_remaining_input_and_truncation(z, oracle):
    d = corpus_small()[30][1]
    c = oracle.deflate(d, level=6)
    out, used, st = z.inflate_batch([c + b"\x01\x02\x03TRAILER"], [len(d)])
    assert out[0] == d and int(used[0]) == len(c)  # trap T14: RemainingInput counts everything after the last EOB byte
    for cut in (1, len(c) // 2, len(c) - 1):
        out, used, st = z.inflate_batch([c[:cut]], [len(d)], raise_on_error=False)
        assert int(st[0]) & 0xFF == 8  # needs input, not a data error
        assert d.startswith(out[0])
    out, used, st = z.inflate_batch([c], [len(d) - 1], raise_on_error=False)
    assert int(st[0]) & 0xFF == 7  # capacity


def test_inflate_error_cases(z):
    # reserved block type 3; stored block with bad NLEN; distance code 30
    cases = {bytes([0x07, 0x00]): 1, bytes([0x01, 0x05, 0x00, 0x00, 0x00]): 2}
    for raw, detail in cases.items():
        out, used, st = z.inflate_batch([raw], [1024], raise_on_error=False)
        assert int(st[0]) & 0xFF == 3 and (int(st[0]) >> 8) == detail, (raw.hex(), st)


def test_inflate_c2_shape(z, oracle):
    from sharpziplib_b200 import datagen
    bufs = [datagen.text_buffer(i, 1 << 20).tobytes() for i in range(8)]
    comp = oracle.batch(0, bufs, level=6, threads=8)
    out, used, st = z.inflate_batch(comp, [len(b) for b in bufs])
    assert out == bufs


# ---- device plans (the benchmark's path) -------------------------------------------------------------------
def test_plans_on_device_tensors(z, oracle):
    import torch
    from sharpziplib_b200 import datagen
    bufs = [datagen.silesia_mix(i, 50000 + 3000 * i).tobytes() for i in range(16)]
    plan = z.DeflatePlan([len(b) for b in bufs], level=6)
    host = np.zeros(plan.in_bytes, dtype=np.uint8)
    for o, b in zip(plan.in_offsets, bufs):
        host[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    d_in = torch.from_numpy(host).cuda()
    d_out = torch.empty(plan.out_bytes, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(len(bufs), dtype=torch.int64, device="cuda")
    d_st = torch.zeros(len(bufs), dtype=torch.int32, device="cuda")
    plan.run(d_in, d_out, d_len, d_st)
    plan.run(d_in, d_out, d_len, d_st)  # idempotent
    torch.cuda.synchronize()
    lens = d_len.cpu().numpy()
    out = d_out.cpu().numpy()
    comp = [out[o:o + l].tobytes() for o, l in zip(plan.out_offsets, lens)]
    assert comp == [oracle.deflate(b, level=6) for b in bufs]
    assert plan.launches >= 6
    ip = z.InflatePlan([len(c) for c in comp], [len(b) for b in bufs])
    hin = np.zeros(ip.in_bytes, dtype=np.uint8)
    for o, c in zip(ip.in_offsets, comp):
        hin[o:o + len(c)] = np.frombuffer(c, dtype=np.uint8)
    di = torch.from_numpy(hin).cuda()
    do = torch.empty(ip.out_bytes, dtype=torch.uint8, device="cuda")
    dl = torch.zeros(len(bufs), dtype=torch.int64, device="cuda")
    ds = torch.zeros(len(bufs), dtype=torch.int32, device="cuda")
    du = torch.zeros(len(bufs), dtype=torch.int64, device="cuda")
    ip.run(di, do, dl, ds, None, du)
    torch.cuda.synchronize()
    o2 = do.cpu().numpy()
    assert [o2[o:o + l].tobytes() for o, l in zip(ip.out_offsets, dl.cpu().numpy())] == bufs
    assert ds.cpu().numpy().tolist() == [0] * len(bufs)


# ---- streaming handles and stream adapters (the reference's own test shapes) ------------------------------
@pytest.mark.parametrize("level", [0, 1, 5, 6, 9])
@pytest.mark.parametrize("zlib_wrap", [True, False])
def test_inflate_deflate_roundtrip_like_reference(z, oracle, level, zlib_wrap):
    """InflaterDeflaterTests.InflateDeflateZlib / NonZlib (:157-162, :226-231): 100000 random bytes,
    Write(all) -> Flush() -> Finish(), read back through InflaterInputStream."""
    original = oracle.dotnet_random_bytes(5, 100000).tobytes()  # Utils.GetDummyBytes(100000): new Random(5).NextBytes
    ms = io.BytesIO()
    out = z.DeflaterOutputStream(ms, z.Deflater(level, not zlib_wrap))
    out.IsStreamOwner = False
    out.Write(original)
    out.Flush()
    out.Finish()
    comp = ms.getvalue()
    assert comp == oracle.deflate(original, level=level, nowrap=not zlib_wrap, pattern=1)
    ins = z.InflaterInputStream(io.BytesIO(comp), z.Inflater(not zlib_wrap))
    assert ins.read() == original


def test_deflater_handle_members(z, oracle):
    d = corpus_small()[40][1]
    df = z.Deflater(6, True)
    assert df.IsNeedingInput and not df.IsFinished and df.GetLevel() == 6
    df.SetInput(d[:1000])
    buf = bytearray(512)
    assert df.Deflate(buf) == 0 and df.IsNeedingInput  # "need more input" is the normal answer (Deflater.cs:480-484)
    df.SetInput(d[1000:])
    df.Finish()
    out = b""
    while not df.IsFinished:
        n = df.Deflate(buf)
        assert n > 0
        out += bytes(buf[:n])
    assert out == oracle.deflate(d, level=6)
    assert df.TotalIn == len(d) and df.TotalOut == len(out)
    df.Reset()
    df.SetLevel(9)
    df.SetInput(d)
    df.Finish()
    out = b""
    while not df.IsFinished:
        n = df.Deflate(buf)
        out += bytes(buf[:n])
    assert out == oracle.deflate(d, level=9)
    for lvl in (0, 1, 3):
        df2 = z.Deflater(lvl, False)
        df2.SetInput(d)
        df2.Finish()
        out = b""
        while not df2.IsFinished:
            n = df2.Deflate(buf)
            out += bytes(buf[:n])
        assert out == oracle.deflate(d, level=lvl, nowrap=False)


def test_inflater_handle_members(z, oracle):
    d = corpus_small()[41][1]
    c = oracle.deflate(d, level=6, nowrap=False)
    inf = z.Inflater(False)
    assert inf.IsNeedingInput
    inf.SetInput(c[:100])
    buf = bytearray(1 << 16)
    got = b""
    n = inf.Inflate(buf)
    got += bytes(buf[:n])
    assert inf.IsNeedingInput and not inf.IsFinished
    inf.SetInput(c[100:] + b"EXTRA")
    while not inf.IsFinished:
        n = inf.Inflate(buf)
        if n == 0:
            break
        got += bytes(buf[:n])
    assert got == d and inf.IsFinished
    assert inf.RemainingInput == 5 and inf.TotalIn == len(c) and inf.TotalOut == len(d)
    assert inf.Adler == zlib.adler32(d)
    bad = bytearray(c)
    bad[-1] ^= 0xFF
    inf.Reset()
    inf.SetInput(bytes(bad))
    with pytest.raises(z.SharpZipBaseException):
        while True:
            if inf.Inflate(buf) == 0:
                break
    inf2 = z.Inflater(False)
    inf2.SetInput(b"\x79\x9c\x03\x00")
    with pytest.raises(z.SharpZipBaseException):
        inf2.Inflate(buf)  # "Header checksum illegal"


def test_gzip_streams(z):
    import gzip
    from sharpziplib_b200 import datagen
    d = datagen.gen_log(300000, 11).tobytes()
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.ModifiedTime = 1577836800
    for i in range(0, len(d), 65536):
        g.Write(d[i:i + 65536])
    g.Finish()
    blob = ms.getvalue()
    assert blob[:10] == bytes([0x1F, 0x8B, 8, 0, 0x00, 0xE1, 0x0B, 0x5E, 0, 255])  # trap T15: XFL 0, OS 255
    assert gzip.decompress(blob) == d
    assert z.GZipInputStream(io.BytesIO(blob)).read() == d
    assert z.GZipInputStream(io.BytesIO(blob + blob)).read() == d + d  # multi-member


# ---- randomised shapes ------------------------------------------------------------------------------------
def test_fuzz_deflate_inflate_against_oracle(z, oracle):
    """seeded random batches: ragged sizes around every block / window / round boundary, all levels and strategies, the three
    wrappers; every stream must equal the oracle's bytes and must come back through the device inflater unchanged"""
    import random
    rnd = random.Random(20240917)
    edges = [0, 1, 2, 3, 4, 31, 32, 33, 257, 258, 259, 1023, 1024, 1025, 16383, 16384, 16385, 32505, 32506, 32507, 32767, 32768,
             32769, 65273, 65274, 65535, 65536, 65537, 98041, 98042, 131071, 131072, 200000]
    for trial in range(6):
        n = rnd.randrange(3, 12)
        bufs = []
        for _ in range(n):
            size = rnd.choice(edges) if rnd.random() < 0.6 else rnd.randrange(0, 150000)
            cls = rnd.randrange(8)
            b = datagen.silesia_mix(cls, max(size, 1), config=rnd.randrange(1, 9)).tobytes()[:size]
            if rnd.random() < 0.2 and size:
                b = bytes([b[0]]) * size            # a single-byte run: nice-length exits, maximal matches
            bufs.append(b)
        level = rnd.choice([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 6, 9])
        strategy = rnd.choice([0, 0, 1, 2])
        wrap = rnd.choice([0, 1])
        end_mode = rnd.choice([0, 0, 1])
        outs, _ = z.deflate_batch(bufs, level=level, strategy=strategy, wrap=wrap, end_mode=end_mode)
        want = [oracle.deflate(b, level=level, strategy=strategy, nowrap=(wrap == 0), pattern=(1 if end_mode else 0)) for b in bufs]
        for i, (g, w) in enumerate(zip(outs, want)):
            assert g == w, (trial, i, len(bufs[i]), level, strategy, wrap, end_mode)
        raw = [o[2:-4] if wrap else o for o in outs]
        back, used, st = z.inflate_batch(raw, [len(b) + 16 for b in bufs])
        assert [int(x) for x in st] == [0] * n
        for i, b in enumerate(bufs):
            assert back[i] == b and int(used[i]) == len(raw[i]), (trial, i)


# ---- framing on the device: zlib / gzip headers and trailers around inflate plans ---------------------------------
def _gzip_member(data, level=6, fname=None, extra=None, comment=None, hcrc=False, mtime=0):
    """a gzip member as GZipOutputStream would frame it, with optional header fields; FHCRC written the way the reference
    READS it (high byte first, GzipInputStream.cs:286-306)"""
    import struct
    flags = (4 if extra is not None else 0) | (8 if fname is not None else 0) | (16 if comment is not None else 0) | (2 if hcrc else 0)
    h = bytearray([0x1F, 0x8B, 8, flags]) + struct.pack("<I", mtime) + bytes([0, 255])
    if extra is not None:
        h += struct.pack("<H", len(extra)) + extra
    if fname is not None:
        h += fname + b"\0"
    if comment is not None:
        h += comment + b"\0"
    if hcrc:
        c = zlib.crc32(bytes(h)) & 0xFFFF
        h += bytes([c >> 8, c & 0xFF])
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    raw = co.compress(data) + co.flush()
    return bytes(h) + raw + struct.pack("<II", zlib.crc32(data) & 0xFFFFFFFF, len(data) & 0xFFFFFFFF), len(h)


def test_inflate_zlib_framing_on_device(z, oracle):
    bufs = [d for _, d in corpus_small() if len(d) >= 10][:12] + [b"", datagen.gen_text(300000, 3).tobytes()]
    comp = [oracle.deflate(b, level=6, nowrap=False) for b in bufs]
    out, used, st, chk = z.inflate_batch(comp, [len(b) + 8 for b in bufs], wrap=1, return_checks=True)
    assert [int(x) for x in st] == [0] * len(bufs)
    for i, b in enumerate(bufs):
        assert out[i] == b and int(used[i]) == len(comp[i]) and int(chk[i]) == zlib.adler32(b), i
    # trailing bytes are not consumed; a wrong trailer, header check and method are the reference's errors
    c = comp[3]
    cases = [(c + b"xyz", 0, 0, len(c)), (c[:-1] + bytes([c[-1] ^ 1]), 3, 11, None), (bytes([c[0], c[1] ^ 1]) + c[2:], 3, 19, None),
             (bytes([0x79, 0x9C ^ 0x1F]) + c[2:], 3, None, None), (c[:-2], 8, 0, len(c) - 2), (c[:1], 8, 0, None)]
    for blob, code, det, want_used in cases:
        o, u, s = z.inflate_batch([blob], [len(bufs[3]) + 8], wrap=1, raise_on_error=False)
        assert int(s[0]) & 0xFF == code, (code, int(s[0]))
        if det is not None:
            assert int(s[0]) >> 8 == det
        if want_used is not None:
            assert int(u[0]) == want_used
    with pytest.raises(z.SharpZipBaseException, match="Adler chksum"):
        z.inflate_batch([c[:-1] + bytes([c[-1] ^ 1])], [len(bufs[3]) + 8], wrap=1)


def test_inflate_gzip_framing_on_device(z):
    data = datagen.gen_text(200000, 21).tobytes()
    variants = [dict(), dict(fname=b"file.txt"), dict(extra=b"\x01\x02abcd"), dict(comment=b"hello"), dict(hcrc=True),
                dict(fname=b"n", extra=b"", comment=b"c", hcrc=True, mtime=123456789)]
    members = [_gzip_member(data[: 1000 * (i + 1) * 37], **v) for i, v in enumerate(variants)]
    blobs = [m for m, _ in members]
    out, used, st, chk = z.inflate_batch(blobs, [len(data) + 8] * len(blobs), wrap=2, return_checks=True)
    assert [int(x) for x in st] == [0] * len(blobs)
    for i in range(len(blobs)):
        want = data[: 1000 * (i + 1) * 37]
        assert out[i] == want and int(used[i]) == len(blobs[i]) and int(chk[i]) == zlib.crc32(want), i
    # two members back to back: the first run stops behind the first footer, the rest starts a new header there
    two = blobs[1] + blobs[2]
    o, u, s = z.inflate_batch([two], [len(data) + 8], wrap=2)
    assert int(s[0]) == 0 and int(u[0]) == len(blobs[1]) and o[0] == data[:74000]
    o, u, s = z.inflate_batch([two[int(u[0]):]], [len(data) + 8], wrap=2)
    assert int(s[0]) == 0 and o[0] == data[:111000]
    # every header / footer error of GZipInputStream (detail codes in INTEGRATION.md)
    g, hl = members[5]
    bad = lambda i, v: g[:i] + bytes([v]) + g[i + 1:]
    cases = [(bad(0, 0x1E), 3, 14), (bad(1, 0x8C), 3, 15), (bad(2, 7), 3, 16), (bad(3, g[3] | 0x20), 3, 17),
             (bad(hl - 1, g[hl - 1] ^ 1), 3, 18), (bad(len(g) - 8, g[-8] ^ 1), 3, 12), (bad(len(g) - 1, g[-1] ^ 1), 3, 13),
             (g[:-3], 8, 0), (g[:hl - 1], 8, 0), (g[:5], 8, 0)]
    for blob, code, det in cases:
        o, u, s = z.inflate_batch([blob], [len(data) + 8], wrap=2, raise_on_error=False)
        assert (int(s[0]) & 0xFF, int(s[0]) >> 8) == (code, det), (code, det, int(s[0]))


def test_inflate_raw_with_crc_for_zip_entries(z, oracle):
    bufs = [datagen.silesia_mix(c, 90000 + 1111 * c, config=4).tobytes() for c in range(6)] + [b""]
    comp = [oracle.deflate(b, level=9) for b in bufs]
    out, used, st, chk = z.inflate_batch(comp, [len(b) + 8 for b in bufs], wrap=3, return_checks=True)
    assert [int(x) for x in st] == [0] * len(bufs)
    for i, b in enumerate(bufs):
        assert out[i] == b and int(chk[i]) == zlib.crc32(b) and int(used[i]) == len(comp[i]), i


def test_zip_entry_batch_roundtrip_through_a_real_container(z, oracle):
    """f2: entry payloads compressed in one batch (raw stream + CRC-32 + size = a passthrough entry); assembled into a
    minimal container here and read back by Python's zipfile, then through the device read path"""
    import struct
    import zipfile
    names = ["a.txt", "dir/b.bin", "empty", "c.log"]
    datas = [datagen.gen_text(70000, 1).tobytes(), datagen.silesia_mix(5, 123457, config=2).tobytes(), b"",
             datagen.gen_log(200000, 9).tobytes()]
    ents = z.zip_entries(datas, level=6)
    for e, d in zip(ents, datas):
        assert e["raw"] == oracle.deflate(d, level=6) and e["crc"] == zlib.crc32(d) and e["size"] == len(d)
    blob, central = bytearray(), bytearray()
    for name, e in zip(names, ents):
        n = name.encode()
        off = len(blob)
        blob += struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, 0, 8, 0, 0x21, e["crc"], len(e["raw"]), e["size"], len(n), 0) + n + e["raw"]
        central += struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 20, 20, 0, 8, 0, 0x21, e["crc"], len(e["raw"]), e["size"], len(n), 0, 0,
                               0, 0, 0, off) + n
    cd_off = len(blob)
    blob += central + struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, len(names), len(names), len(central), cd_off, 0)
    with zipfile.ZipFile(io.BytesIO(bytes(blob))) as zf:
        assert zf.testzip() is None
        for name, d in zip(names, datas):
            assert zf.read(name) == d
    back = z.unzip_entries([e["raw"] for e in ents], [e["size"] for e in ents], [e["crc"] for e in ents])
    assert back == datas
    with pytest.raises(z.SharpZipBaseException):
        z.unzip_entries([ents[0]["raw"]], [ents[0]["size"]], [ents[0]["crc"] ^ 1])


# ---- the reference's own GZip stream tests, against the mirror (test/ICSharpCode.SharpZipLib.Tests/GZip/GZipTests.cs) ----
def _dummy_bytes(size, seed=1):
    return datagen.Rng(1000 + seed).bytes(size).tobytes()


def test_gzip_reference_tests_delayed_header(z):
    """DelayedHeaderWriteNoData / FlushNoData / WithData / FlushWithData (:65-160)"""
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    assert len(ms.getvalue()) == 0
    g.Close()
    assert len(ms.getvalue()) != 0
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.Flush()  # issue 382: flushing before anything was written
    g.Close()
    assert z.GZipInputStream(io.BytesIO(ms.getvalue())).read() == b""
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.WriteByte(45)
    assert len(ms.getvalue()) == 10  # the header, with one byte in the compression pipeline
    g.Close()
    assert z.GZipInputStream(io.BytesIO(ms.getvalue())).read() == bytes([45])
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.Flush()
    g.WriteByte(45)  # input after a sync flush
    g.Close()
    assert z.GZipInputStream(io.BytesIO(ms.getvalue())).read() == bytes([45])


def test_gzip_reference_tests_reader(z):
    """ZeroLengthInputStream (:166), DoubleFooter (:241), TrailingGarbage (:291), FlushToUnderlyingStream (:343),
    OriginalFilename (:480)"""
    assert z.GZipInputStream(io.BytesIO(b"")).ReadByte() == -1
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.Finish()
    length = len(ms.getvalue())
    g.Close()  # a second Finish must not write a second footer
    assert len(ms.getvalue()) == length
    buf = _dummy_bytes(100000, 3)
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.Write(buf)
    g.Flush()
    g.Finish()
    garbage = _dummy_bytes(4096, 4)
    r = z.GZipInputStream(io.BytesIO(ms.getvalue() + garbage))
    got = bytearray(len(buf))
    idx = 0
    while idx < len(got):
        n = r.Read(got, idx, len(got) - idx)
        if n <= 0:
            break
        idx += n
    assert idx == len(buf) and bytes(got) == buf and r.Read(bytearray(16), 0, 16) == 0
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.Write(buf)
    g.Flush()  # flushed, not finished: everything written so far must be readable
    r = z.GZipInputStream(io.BytesIO(ms.getvalue()))
    got, idx = bytearray(len(buf)), 0
    try:
        while idx < len(got):
            n = r.Read(got, idx, len(got) - idx)
            if n <= 0:
                break
            idx += n
        r.Read(bytearray(1), 0, 1)
        raised = False
    except z.SharpZipBaseException:
        raised = True  # "unexpected EOF" once all data has been read
    assert idx == len(buf) and bytes(got) == buf and raised
    ms = io.BytesIO()
    g = z.GZipOutputStream(ms)
    g.IsStreamOwner = False
    g.FileName = "/path/to/file.ext"
    g.Write(b"FileContents")
    g.Flush()
    g.Finish()
    r = z.GZipInputStream(io.BytesIO(ms.getvalue()))
    assert r.read(12) == b"FileContents" and r.GetFilename() == "file.ext"
