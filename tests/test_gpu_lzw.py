"""GPU tier: LZW (.Z) decompression (b200z_lzw.cu) against the LzwInputStream restatement of tests/cpu_model/lzw_model.cpp,
on streams of its compress(1)-format encoder and on hand-built corrupt streams."""
import hashlib
import io
import os

import numpy as np
import pytest

import lzw_ref as R
from lzw_quirks import QUIRKS

pytestmark = pytest.mark.gpu


def _text(n, seed=1):
    rng = np.random.default_rng(seed)
    words = [b"alpha", b"beta", b"gamma", b"delta", b"lzw", b"compress", b"\n", b" ", b"2009", b"GNSS"]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(len(words)))]
    return bytes(out[:n])


def _check(z, streams, caps=None):
    outs, status, value = z.lzw_batch(streams, caps)
    for i, s in enumerate(streams):
        r = R.decode(s, out_chunk=1) if len(s) < 4096 else R.decode(s)
        st = int(status[i])
        assert outs[i] == r.out[:len(outs[i])] and len(outs[i]) == r.decoded, (i, len(outs[i]), r)
        if r.kind == 0:
            assert st == 0, (i, st)
        elif r.kind == 6:  # the failure site: the header's tables, ResetBuf, the string tables
            assert st & 0xFF == 4 and st >> 8 == r.a, (i, st, r)
        else:
            assert st & 0xFF == 3, (i, st, r)
            assert str(z.lzw.error_for(st, int(value[i]))) == r.message
    return outs, status


@pytest.mark.parametrize("block", [True, False])
def test_max_bits_9_to_16(z, block):
    d = _text(300000) + bytes(range(256)) * 40 + bytes(20000)
    _check(z, [R.encode(d, mb, block) for mb in range(9, 17)])


@pytest.mark.parametrize("k", [1, 2, 255, 4096])
def test_clear_every_k_codes(z, k):
    d = _text(100000, seed=k)
    _check(z, [R.encode(d, mb, True, clear_every=k) for mb in (9, 12, 16)])


def test_long_table_full_epochs(z):
    rng = np.random.default_rng(5)
    d = bytes(rng.integers(0, 16, 3 << 20, dtype=np.uint8))
    _check(z, [R.encode(d, mb, block, ratio_clear=False) for mb in (12, 16) for block in (True, False)])


def test_silesia_mix_classes(z):
    from sharpziplib_b200 import datagen
    streams = [R.encode(datagen.silesia_mix(i, 256 << 10).tobytes(), 16) for i in range(1024)]
    outs, _ = _check(z, streams[:64])
    outs, status, _ = z.lzw_batch(streams)
    assert not status.any()
    for i in range(0, 1024, 37):
        assert outs[i] == datagen.silesia_mix(i, 256 << 10).tobytes()


def test_random_bytes_and_zeros(z):
    rng = np.random.default_rng(9)
    rnd = bytes(rng.integers(0, 256, 1 << 20, dtype=np.uint8))
    zeros = bytes(64 << 20)
    outs, _ = _check(z, [R.encode(rnd, 16), R.encode(zeros, 16), R.encode(zeros, 16, False)])
    assert len(R.encode(rnd, 16)) > len(rnd)


@pytest.mark.skipif(os.environ.get("B200Z_EMU_ORDER") is not None, reason="2 GiB of output: device only")
def test_zeros_with_a_full_table(z):
    import lzw_quirks
    n = 65280 * 65281 // 2 + 5 * 65280 + 777  # the table fills; then five strings of 65280 bytes and a short one
    s = lzw_quirks.zeros_stream(n)
    outs, status, _ = z.lzw_batch([s], [n])
    assert status[0] == 0 and len(outs[0]) == n and outs[0].count(0) == n
    p = z.LzwPlan([len(s)], [n])
    _plan_run(p, [s])
    assert p.stats()["longest"] == 65280


def test_quirk_streams(z):
    _check(z, [s for _, s in QUIRKS])


def test_nomem_reports_the_size_and_retries(z):
    d = _text(50000)
    s = R.encode(d, 14)
    outs, status, value = z.lzw_batch([s], [100])
    assert outs[0] == d and status[0] == 0
    L = z.lib()
    import ctypes as C
    ins = np.frombuffer(s, np.uint8)
    out = np.zeros(101, np.uint8)
    ol, iu, vv, st = (np.zeros(1, np.int64), np.zeros(1, np.int64), np.zeros(1, np.uint32), np.zeros(1, np.int32))
    lens, caps = np.array([len(s)], np.int64), np.array([100], np.int64)
    rc = L.b200z_lzw_batch((C.c_void_p * 1)(ins.ctypes.data), lens.ctypes.data, 1, (C.c_void_p * 1)(out.ctypes.data), caps.ctypes.data,
                           ol.ctypes.data, iu.ctypes.data, vv.ctypes.data, st.ctypes.data)
    assert rc == 7 and st[0] == 7 and ol[0] == len(d)


def _plan_run(p, streams, timing=False):
    import torch
    blob = np.zeros(p.in_bytes, np.uint8)
    for i, s in enumerate(streams):
        blob[p.in_offsets[i]:p.in_offsets[i] + len(s)] = np.frombuffer(s, np.uint8)
    n = len(streams)
    t = dict(d_in=torch.from_numpy(blob).cuda(), d_out=torch.zeros(p.out_bytes, dtype=torch.uint8, device="cuda"),
             ol=torch.zeros(n, dtype=torch.int64, device="cuda"), st=torch.zeros(n, dtype=torch.int32, device="cuda"),
             val=torch.zeros(n, dtype=torch.int32, device="cuda"), used=torch.zeros(n, dtype=torch.int64, device="cuda"))
    p.set_timing(timing)
    p.run(t["d_in"], t["d_out"], t["ol"], t["st"], t["val"], t["used"])
    torch.cuda.synchronize()
    return t


def test_plan_run_stats_and_timing(z):
    d = _text(200000)
    streams = [R.encode(d, 16, True, clear_every=5000), R.encode(bytes(100000), 16)]
    p = z.LzwPlan([len(s) for s in streams], [len(d), 100000])
    t = _plan_run(p, streams, timing=True)
    ol, st, used = t["ol"], t["st"], t["used"]
    out = t["d_out"].cpu().numpy()
    assert ol.tolist() == [len(d), 100000] and st.tolist() == [0, 0]
    assert out[p.out_offsets[0]:p.out_offsets[0] + len(d)].tobytes() == d
    assert used.tolist() == [len(streams[0]), len(streams[1])]
    stats = p.stats()
    assert stats["epochs"] >= 3 and stats["longest"] > 400
    assert set(p.timings()) >= {"k_lzw_scan", "k_lzw_jump", "k_lzw_emit"}


def test_pack_refuses_lzw_plans(z):
    import torch
    d = _text(50000)
    streams = [R.encode(d, 14), R.encode(d[:1000], 14)]
    p = z.LzwPlan([len(s) for s in streams], [100, 2000])  # stream 0 does not fit: its out_len is the size it needs
    t = _plan_run(p, streams)
    assert t["st"].tolist() == [7, 0] and t["ol"].tolist() == [len(d), 1000]
    packed = torch.zeros(p.out_bytes, dtype=torch.uint8, device="cuda")
    packed.fill_(0xA5)
    poff = torch.zeros(3, dtype=torch.int64, device="cuda")
    with pytest.raises(z.B200zUnsupported):
        p.pack(t["d_out"], t["ol"], packed, poff)
    torch.cuda.synchronize()
    assert bool((packed == 0xA5).all()) and not poff.any()


def test_pipeline_depth_2_and_multi(z):
    import ctypes as C
    L = z.lib()
    batches = [[R.encode(_text(30000 + 1000 * i, seed=b), 12) for i in range(8)] for b in range(3)]
    lens = np.array([len(s) for s in batches[0]], np.int64)
    caps = np.full(8, 80000, np.int64)
    h = C.c_void_p()
    # every batch must have the plan's lengths: later batches are cut or padded with zero bytes (which decode as more codes;
    # the oracle decodes the same padded streams)
    same = [[s + bytes(int(lens[i]) - len(s)) if len(s) <= lens[i] else s[:lens[i]] for i, s in enumerate(b)] for b in batches]
    assert L.b200z_lzw_pipeline_create(8, lens.ctypes.data, caps.ctypes.data, 2, C.byref(h)) == 0
    pipe = z.Pipeline(h, 8, 2)
    keep = [[np.frombuffer(s, np.uint8) for s in b] for b in same]
    outs = [[np.zeros(80001, np.uint8) for _ in range(8)] for _ in same]
    pipe.submit(pipe.pointers([a.ctypes.data for a in keep[0]]))
    pipe.submit(pipe.pointers([a.ctypes.data for a in keep[1]]))
    assert pipe.in_flight == 2
    for k in range(3):
        pipe.collect(pipe.pointers([a.ctypes.data for a in outs[k]]), caps, raise_on_error=False)
        if k == 0:
            pipe.submit(pipe.pointers([a.ctypes.data for a in keep[2]]))
        for i in range(8):
            r = R.decode(same[k][i])
            assert outs[k][i][:pipe.out_len[i]].tobytes() == r.out[:pipe.out_len[i]] and pipe.out_len[i] == r.decoded
    pipe.close()
    devs = list(range(z.lib().b200z_device_count()))
    o1, s1, _ = z.lzw_batch(batches[0] * 4, devices=devs)
    assert not s1.any() and o1 == [R.decode(s).out for s in batches[0] * 4]


@pytest.mark.parametrize("chunk", [1, 4096, 1 << 20])
def test_input_stream_reads(z, chunk):
    cases = [R.encode(_text(20000), 13)] + [s for name, s in QUIRKS if name in ("code_gt_free_ent", "truncated_after_pad",
                                                                              "first_code_clear", "bad_magic")]
    for s in cases:
        r = R.decode(s, out_chunk=chunk)
        st = z.LzwInputStream(io.BytesIO(s))
        got = bytearray()
        err = None
        try:
            while True:
                b = bytearray(chunk)
                k = st.Read(b, 0, chunk)
                if k <= 0:
                    break
                got += b[:k]
        except Exception as e:  # noqa: BLE001
            err = e
        assert bytes(got) == r.out
        assert (err is None) == (r.kind == 0)
        if r.kind in R.MESSAGES:
            assert isinstance(err, z.LzwException) and str(err) == r.message


@pytest.mark.skipif(os.environ.get("B200Z_EMU_ORDER") is not None, reason="4 GiB of output: device only")
def test_output_past_4_gib(z):
    import lzw_quirks
    zeros = 4 * (1 << 30) + 12345
    s = lzw_quirks.zeros_stream(zeros)
    outs, status, _ = z.lzw_batch([s], [zeros])
    assert status[0] == 0 and len(outs[0]) == zeros
    assert hashlib.sha256(outs[0]).digest() == hashlib.sha256(bytes(zeros)).digest()
