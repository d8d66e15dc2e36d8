"""GPU tier: the block-parallel inflate pipeline (csrc/b200z_inflate_par.cuh) against the oracle's Inflater, against zlib and
against the serial kernel, through the C-ABI.  What is pinned here: the pipeline really runs (segments found by the block
finder are decoded and joined, nothing handed back), its results -- bytes, TotalOut, RemainingInput, status and detail,
restart points -- equal the serial kernel's on valid, truncated and corrupt streams, and the host-buffer pipelines and
the one-process multi-GPU calls deliver the same bytes."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from helpers import corpus_small
from sharpziplib_b200 import datagen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_plan(z, comp, caps, wrap=0, dict_lens=None, dicts=None, start_bits=None):
    import torch
    plan = z.InflatePlan([len(c) for c in comp], caps, wrap=wrap, dict_lens=dict_lens)
    h = np.zeros(plan.in_bytes, dtype=np.uint8)
    for i, c in enumerate(comp):
        if dicts is not None and dict_lens[i]:
            h[plan.in_offsets[i]:plan.in_offsets[i] + dict_lens[i]] = np.frombuffer(dicts[i][-dict_lens[i]:], dtype=np.uint8)
        o = plan.data_offsets[i]
        h[o:o + len(c)] = np.frombuffer(c, dtype=np.uint8)
    if start_bits is not None:
        plan.set_start_bits(start_bits)
    n = len(comp)
    d_in = torch.from_numpy(h).cuda()
    d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_ck = torch.zeros(n, dtype=torch.int32, device="cuda")
    plan.run(d_in, d_out, d_len, d_st, d_ck, d_used)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    lens = d_len.cpu().numpy()
    res = [out[plan.out_offsets[i]:plan.out_offsets[i] + lens[i]].tobytes() for i in range(n)]
    bits, pos = plan.restart_points()
    stats = plan.stats()
    plan.close()
    return res, d_st.cpu().numpy(), d_used.cpu().numpy(), bits, pos, stats


def _serial(fn, *a, **k):
    """the same call with the serial kernel alone (B200Z_INFLATE=serial is read when a plan is built)"""
    os.environ["B200Z_INFLATE"] = "serial"
    try:
        return fn(*a, **k)
    finally:
        del os.environ["B200Z_INFLATE"]


def test_segments_are_found_and_joined(z, oracle):
    """multi-block streams: the finder's candidates become segments, every stream is resolved by the pipeline itself"""
    bufs = [datagen.text_buffer(i, (1 << 20) - 4097 * i).tobytes() for i in range(6)] + \
           [datagen.silesia_mix(i, 600000 + 12345 * i).tobytes() for i in range(8)]
    comp = [oracle.deflate(b, level=6 if i % 3 else 9) for i, b in enumerate(bufs)]
    res, st, used, bits, pos, stats = _run_plan(z, comp, [len(b) + 7 for b in bufs])
    assert stats["parallel"] == 1 and stats["handed_back"] == 0
    assert stats["segments"] > 2 * len(bufs) and stats["blocks"] >= stats["segments"], stats
    assert res == bufs and not st.any() and [int(u) for u in used] == [len(c) for c in comp]
    res2, st2, used2, bits2, pos2, stats2 = _serial(_run_plan, z, comp, [len(b) + 7 for b in bufs])
    assert stats2["parallel"] == 0 and res2 == res
    assert list(bits) == list(bits2) and list(pos) == list(pos2)  # the restart point: the final block's header


def test_c2_shape_every_stream(z, oracle):
    """config C2 at its full size: 256 x 1 MiB text, every inflated stream compared"""
    bufs = [datagen.text_buffer(i, 1 << 20, config=2).tobytes() for i in range(256)]
    comp = oracle.batch(0, bufs, level=6, threads=16)
    res, st, used, _, _, stats = _run_plan(z, comp, [len(b) for b in bufs])
    assert not st.any() and stats["handed_back"] == 0
    for i in range(256):
        assert res[i] == bufs[i], i
        assert int(used[i]) == len(comp[i])


def test_foreign_streams_stored_static_and_mixed_blocks(z):
    """zlib's streams: stored blocks (level 0), static blocks (tiny inputs, Z_FIXED), sync-flush markers between blocks,
    incompressible data, long runs (distance 1, overlapping copies)"""
    rng = datagen.Rng(77)
    items = []
    text = datagen.gen_text(300000, 5).tobytes()
    items.append(zlib.compress(text, 0)[2:-4])                      # stored blocks only
    co = zlib.compressobj(6, zlib.DEFLATED, -15, 9, zlib.Z_FIXED)
    items.append(co.compress(text[:50000]) + co.flush())            # one long static block
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    parts = b""
    for k in range(0, 200000, 7000):                                # a sync flush (empty stored block) every 7000 bytes
        parts += co.compress(text[k:k + 7000]) + co.flush(zlib.Z_SYNC_FLUSH)
    items.append(parts + co.flush())
    rnd = rng.bytes(400000).tobytes()
    items.append(zlib.compress(rnd, 6)[2:-4])
    runs = (b"\x00" * 70000 + b"ab" * 40000 + bytes(range(256)) * 300 + b"\xff" * 100000)
    items.append(zlib.compress(runs, 9)[2:-4])
    mixed = text[:100000] + rnd[:100000] + runs[:100000] + text[100000:200000]
    items.append(zlib.compress(mixed, 6)[2:-4])
    import random
    random.seed(3)
    toks = [bytes(random.randrange(256) for _ in range(4)) for _ in range(40)]
    dense = b"".join(random.choice(toks) for _ in range(60000))    # thousands of 4..8-byte references per 16 KiB of output
    items.append(zlib.compress(dense, 6)[2:-4])
    items.append(zlib.compress(dense[:50000] + runs[:90000] + dense[50000:150000], 4)[2:-4])
    want = [zlib.decompress(c, -15) for c in items]
    res, st, used, _, _, stats = _run_plan(z, items, [len(w) for w in want])
    assert not st.any() and res == want, st
    assert [int(u) for u in used] == [len(c) for c in items]


def test_errors_and_truncation_match_the_serial_kernel(z, oracle):
    """status | detail << 8, bytes produced, RemainingInput and the restart point on corrupt and truncated streams: the
    pipeline's answers are the serial kernel's (which the round-1 tier pinned against the oracle)"""
    base = datagen.text_buffer(3, 400000).tobytes()
    c = oracle.deflate(base, level=6)
    items, caps = [], []
    for cut in (0, 1, 2, 7, 100, len(c) // 3, len(c) // 2, len(c) - 5, len(c) - 1):
        items.append(c[:cut])
        caps.append(len(base))
    rng = np.random.default_rng(5)
    for k in range(24):                                              # a flipped byte somewhere: error, or other bytes
        pos = int(rng.integers(40, len(c) - 40))
        b = bytearray(c)
        b[pos] ^= 1 << int(rng.integers(0, 8))
        items.append(bytes(b))
        caps.append(len(base) + 70000)
    items += [bytes([0x07, 0x00]), bytes([0x01, 0x05, 0x00, 0x00, 0x00]), bytes([0x05, 0xE0, 0x81, 0x08]) + bytes(40)]
    caps += [1024, 1024, 1024]
    a = _run_plan(z, items, caps)
    b = _serial(_run_plan, z, items, caps)
    assert a[5]["parallel"] == 1 and b[5]["parallel"] == 0
    for i in range(len(items)):
        code = int(a[1][i]) & 0xFF
        assert int(a[1][i]) == int(b[1][i]), (i, int(a[1][i]), int(b[1][i]))
        if code == 7:
            continue  # capacity: only the status is defined
        assert a[0][i] == b[0][i], i
        if code in (0, 8):
            assert int(a[2][i]) == int(b[2][i]) and int(a[3][i]) == int(b[3][i]) and int(a[4][i]) == int(b[4][i]), i
    # the reference's own classification at the end of the input (InflaterHuffmanTree.GetSymbol): truncation is "needs input"
    for i in range(9):
        assert int(a[1][i]) & 0xFF == 8 and base.startswith(a[0][i])


def test_distance_code_30_and_length_code_286(z):
    """static blocks address 32 distance and 288 literal/length codes; 30/31 and 286/287 decode and then fail
    (Inflater.cs:318-326, :351-359, trap T13)"""
    def bits_to_bytes(bits):
        out = bytearray((len(bits) + 7) // 8)
        for i, b in enumerate(bits):
            out[i >> 3] |= b << (i & 7)
        return bytes(out) + bytes(8)

    def code(v, n):  # Huffman codes go most significant bit first
        return [(v >> (n - 1 - i)) & 1 for i in range(n)]
    hdr = [1, 1, 0]  # BFINAL = 1, BTYPE = 1 (static)
    lit_a = code(0x30 + 97, 8)
    len3 = code(1, 7)                       # symbol 257
    dist30 = code(30, 5)
    sym286 = code(0xC0 + (286 - 280), 8)
    res, st, _, _, _, _ = _run_plan(z, [bits_to_bytes(hdr + lit_a + len3 + dist30), bits_to_bytes(hdr + lit_a + sym286)], [64, 64])
    assert int(st[0]) & 0xFF == 3 and int(st[0]) >> 8 == 4, st  # "Illegal rep dist code"
    assert int(st[1]) & 0xFF == 3 and int(st[1]) >> 8 == 3, st  # "Illegal rep length code"
    assert res[0] == b"a" and res[1] == b"a"


def test_dictionaries_start_bits_and_framing(z, oracle):
    """preset dictionary (window image in front of the stream), a stream that starts inside a byte, zlib and gzip framing"""
    d = datagen.text_buffer(9, 300000).tobytes()
    dic = d[:20000]
    co = zlib.compressobj(6, zlib.DEFLATED, -15, zdict=dic)
    c = co.compress(d[20000:]) + co.flush()
    res, st, used, _, _, stats = _run_plan(z, [c, c], [len(d), len(d)], dict_lens=[len(dic), 1000], dicts=[dic, dic])
    assert int(st[0]) == 0 and res[0] == d[20000:]
    assert res[1] != res[0]  # only the last 1000 dictionary bytes: the rest of the window reads as zeros (trap T13), no error
    # start inside a byte: 3 junk bits in front of the stream
    raw = oracle.deflate(d, level=6)
    v = int.from_bytes(raw, "little") << 3 | 5
    shifted = v.to_bytes(len(raw) + 1, "little")
    res, st, used, bits, pos, _ = _run_plan(z, [shifted], [len(d)], start_bits=[3])
    assert int(st[0]) == 0 and res[0] == d
    zl, gz = zlib.compress(d, 6), None
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    gz = co.compress(d) + co.flush()
    res, st, used, _, _, _ = _run_plan(z, [zl, zl[:-1] + bytes([zl[-1] ^ 1])], [len(d)] * 2, wrap=1)
    assert int(st[0]) == 0 and res[0] == d and int(used[0]) == len(zl)
    assert int(st[1]) & 0xFF == 3 and int(st[1]) >> 8 == 11  # "Adler chksum doesn't match"
    res, st, used, _, _, _ = _run_plan(z, [gz + b"tail"], [len(d)], wrap=2)
    assert int(st[0]) == 0 and res[0] == d and int(used[0]) == len(gz)


def test_many_tiny_blocks_are_handed_back_and_still_right(z):
    """thousands of empty blocks exhaust the round pool: the stream goes to the serial kernel (handed_back) -- same bytes"""
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    parts = b""
    for k in range(4000):
        parts += co.compress(b"x%d" % k) + co.flush(zlib.Z_FULL_FLUSH)
    parts += co.flush()
    want = zlib.decompress(parts, -15)
    text = datagen.text_buffer(1, 200000).tobytes()
    good = zlib.compress(text, 6)[2:-4]
    res, st, used, _, _, stats = _run_plan(z, [parts, good], [len(want), len(text)])
    assert not st.any() and res == [want, text]
    assert stats["handed_back"] >= 1


def test_host_pipelines_and_gzip_writer(z, oracle):
    """b200z_pipeline_*: depth-2 submit / collect on pageable host memory; wrap = GZIP writes GZipOutputStream's bytes"""
    import ctypes as C
    bufs = [np.frombuffer(datagen.silesia_mix(i, 100000 + 999 * i).tobytes(), dtype=np.uint8).copy() for i in range(12)]
    lens = [b.size for b in bufs]
    P = z.Pipeline
    pipe = P.deflate(lens, level=6, wrap=2, depth=2)
    caps = np.array([z.lib().b200z_deflate_bound(n) + 64 for n in lens], dtype=np.int64)
    outs = [np.zeros(int(c), dtype=np.uint8) for c in caps]
    inp, outp = P.pointers([b.ctypes.data for b in bufs]), P.pointers([o.ctypes.data for o in outs])
    with pytest.raises(Exception):
        pipe.collect(outp, caps)               # nothing submitted: InvalidOperation
    pipe.submit(inp)
    pipe.submit(inp)
    with pytest.raises(Exception):
        pipe.submit(inp)                       # depth 2: two batches in flight
    for _ in range(2):
        pipe.collect(outp, caps)
        for i, b in enumerate(bufs):
            gz = outs[i][:pipe.out_len[i]].tobytes()
            raw = oracle.deflate(b.tobytes(), level=6)
            assert gz[:10] == bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF]) and gz[10:-8] == raw  # trap T15
            assert int.from_bytes(gz[-8:-4], "little") == zlib.crc32(b.tobytes()) and int.from_bytes(gz[-4:], "little") == b.size
            assert zlib.decompress(gz, 31) == b.tobytes()
    pipe.close()
    comp = [np.frombuffer(oracle.deflate(b.tobytes(), level=6), dtype=np.uint8).copy() for b in bufs]
    ip = P.inflate([c.size for c in comp], lens, depth=2)
    backs = [np.zeros(n, dtype=np.uint8) for n in lens]
    icaps = np.array(lens, dtype=np.int64)
    ip.submit(P.pointers([c.ctypes.data for c in comp]))
    ip.collect(P.pointers([b.ctypes.data for b in backs]), icaps)
    assert all(np.array_equal(a, b) for a, b in zip(backs, bufs)) and [int(u) for u in ip.in_used] == [c.size for c in comp]
    ip.close()
    # the batch calls keep their pipeline between calls (same shape: nothing is allocated again)
    for _ in range(3):
        outs2, _ = z.deflate_batch([b.tobytes() for b in bufs], level=6)
        assert outs2 == [c.tobytes() for c in comp]
    z.lib().b200z_release_cached()
    del C


def test_one_process_several_devices(z, oracle):
    """b200z_*_batch_multi: the batch is cut by bytes, every range runs on its device's pipeline, all at the same time.  On
    a one-GPU box the list names the same device twice (two pipelines side by side): the code path is the same."""
    import torch
    ndev = z.lib().b200z_device_count()
    assert ndev == torch.cuda.device_count() >= 1
    devices = list(range(ndev)) if ndev > 1 else [0, 0, 0]
    bufs = [datagen.silesia_mix(i, 30000 + 7000 * (i % 5)).tobytes() for i in range(23)]
    refs = [oracle.deflate(b, level=6) for b in bufs]
    outs, _ = z.deflate_batch(bufs, level=6, devices=devices)
    assert outs == refs
    back, used, st = z.inflate_batch(refs, [len(b) for b in bufs], devices=devices)
    assert back == bufs and not np.any(st)
    outs, _ = z.deflate_batch(bufs[:2], level=6, devices=devices)  # fewer streams than devices: empty ranges
    assert outs == refs[:2]
    z.lib().b200z_release_cached()
    z.init(0)


def _mix64(i):
    return datagen.silesia_mix(i, 64 << 20, config=5)


def test_large_streams(z, oracle):
    """one 256 MiB stream and four 64 MiB streams through deflate (chunked parse) and inflate (hundreds of segments each):
    a checksum of checksums instead of byte lists (size-independent properties)"""
    import hashlib
    big = datagen.log_stream(256 << 20).tobytes()
    outs, chk = z.deflate_batch([big], level=6, wrap=3)
    assert int(chk[0]) == zlib.crc32(big)
    assert hashlib.sha256(zlib.decompress(outs[0], -15)).digest() == hashlib.sha256(big).digest()
    back, used, st = z.inflate_batch(outs, [len(big)])
    assert int(st[0]) == 0 and int(used[0]) == len(outs[0])
    assert hashlib.sha256(back[0]).digest() == hashlib.sha256(big).digest()
    ref = oracle.deflate(big[:32 << 20], level=6)       # the oracle on a prefix stream of its own (32 MiB: seconds)
    outs32, _ = z.deflate_batch([big[:32 << 20]], level=6)
    assert outs32[0] == ref
    del big, back
    from concurrent.futures import ProcessPoolExecutor
    with ProcessPoolExecutor(max_workers=4) as ex:  # (the generators are single-threaded numpy: a minute per 64 MiB)
        four = [a.tobytes() for a in ex.map(_mix64, range(4))]
    outs, _ = z.deflate_batch(four, level=6)
    back, used, st = z.inflate_batch(outs, [len(b) for b in four])
    assert not np.any(st)
    for a, b in zip(back, four):
        assert hashlib.sha256(a).digest() == hashlib.sha256(b).digest()


def test_bench_c4_c5_modes_run_small():
    """bench.py --config c4 / c5 (--small): one JSON line each, parity flags set"""
    import json
    for cfg in ("c4", "c5"):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--config", cfg, "--small", "--steps", "2"],
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        d = json.loads(r.stdout.strip().splitlines()[-1])
        if cfg == "c4":
            assert d["parity_whole_stream_vs_oracle"] and d["crc_ok"] and d["isize_ok"] and d["inflates_to_input"] and d["header_ok"], d
        else:
            assert d["all_parity"] and len(d["points"]) >= 18, d
    assert corpus_small()


def test_bench_dump_outputs(tmp_path):
    """bench.py --dump-outputs: the last timed step's outputs as float .npy files, within 64 MB, equal to what the oracle and
    the generator say they are"""
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--small", "--steps", "2", "--warmup", "1",
                        "--dump-outputs", str(tmp_path)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert json.loads(r.stdout.strip().splitlines()[-1])["steps"] == 2
    a = {f[:-4]: np.load(os.path.join(tmp_path, f)) for f in os.listdir(tmp_path)}
    assert sum(os.path.getsize(os.path.join(tmp_path, f)) for f in os.listdir(tmp_path)) <= 64 << 20
    assert all(v.dtype in (np.float32, np.float64) for v in a.values())
    assert not a["deflate_status"].any() and not a["inflate_status"].any()
    assert (a["inflate_out_len"] == 1 << 20).all()
    i = int(a["inflate_sample_index"][0])
    orig = datagen.text_buffer(i, 1 << 20, config=2).tobytes()
    assert a["inflate_out_crc32"][i] == zlib.crc32(orig)
    assert bytes(a["inflate_sample_bytes"][:1 << 20].astype(np.uint8)) == orig
    j = int(a["deflate_sample_index"][0])
    comp = bytes(a["deflate_sample_bytes"][:int(a["deflate_out_len"][j])].astype(np.uint8))
    assert zlib.crc32(comp) == a["deflate_out_crc32"][j]
    assert zlib.decompress(comp, -15) == datagen.silesia_mix(j, 262144, config=3).tobytes()
