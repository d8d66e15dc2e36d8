"""GPU tier: the CRC-32 / Adler-32 kernel (b200z_checksum.cu) against plain references (tests/checksum_ref.py) at the
lengths, alignments, seeds and sizes where a tile-parallel combination goes wrong: every length up to two chunks, every
chunk and tile edge of the first three tiles, contents that make the Adler sums largest (all 0xFF) or every chunk's partial
equal (period 128), running values as seeds, tiles laid over a capacity and skipped on the device, and streams past 4 GiB.

Every entry point that reaches the kernel is covered: Crc32 / Adler32 (host buffers), b200z_checksum_batch_device,
deflate plans (tiles with multipliers made on the host) and inflate plans (tiles over the output capacity, multipliers made
on the device from the real length).  Tests whose name holds "emu" are small enough for the CUDA emulator; the CPU tier
runs them there.  The cases past 4 GiB check free device and host memory first and skip, saying why, when it is short."""
import gc
import hashlib
import random
import struct
import time
import zlib

import numpy as np
import pytest

from checksum_ref import check_ref
from sharpziplib_b200 import datagen
from test_gpu_inflate_parallel import _serial

pytestmark = pytest.mark.gpu

TILE, CHUNK = 32768, 128  # kCkTile, kCkChunk (b200z_crc.cuh)
BIG, GiB, MiB = 1 << 32, 1 << 30, 1 << 20
EDGE_LENS = list(range(261)) + sorted({TILE * k + d for k in (1, 2, 3) for d in (-129, -128, -1, 0, 1, 127, 128, 129)})
FILLS = ("zeros", "ff", "random", "period128")
KINDS = pytest.mark.parametrize("kind", [0, 1], ids=["crc32", "adler32"])
WRAP_ZLIB, WRAP_GZIP, WRAP_RAW_CRC32 = 1, 2, 3
D_ADLER, D_GZIP_CRC = 11, 12  # status detail: "Adler chksum doesn't match", "GZIP crc sum mismatch"
GZIP_HEADER = bytes([0x1F, 0x8B, 8, 0, 0, 0, 0, 0, 0, 0xFF])


def fill(name, n, seed=1):
    if name == "zeros":
        return np.zeros(n, np.uint8)
    if name == "ff":
        return np.full(n, 0xFF, np.uint8)
    if name == "random":
        return datagen.Rng(seed).bytes(n)
    return np.resize(datagen.Rng(seed + 1000).bytes(CHUNK), n)  # period 128: every full chunk has the same partial


def _new(z, kind):
    return z.Crc32() if kind == 0 else z.Adler32()


def _seed(rnd, kind):
    """a random running value: any 32 bits for CRC-32, both halves below 65521 for Adler-32"""
    if kind == 0:
        return rnd.getrandbits(32)
    return (rnd.randrange(65521) << 16) | rnd.randrange(65521)


# ---- Crc32 / Adler32 on host buffers ------------------------------------------------------------------------------------
@KINDS
@pytest.mark.parametrize("content", FILLS)
def test_emu_host_every_edge_length(z, kind, content):
    """every length 0-260 and 32768 k + {-129, -128, -1, 0, 1, 127, 128, 129}, k = 1..3"""
    buf = fill(content, EDGE_LENS[-1])
    for n in EDGE_LENS:
        c = _new(z, kind)
        c.Update(buf[:n])
        assert c.Value == check_ref(kind, buf[:n]), (content, n, hex(c.Value))


@KINDS
@pytest.mark.parametrize("content", FILLS)
def test_host_five_mib(z, kind, content):
    n = (5 << 20) + 7
    buf = fill(content, n)
    c = _new(z, kind)
    c.Update(buf)
    assert c.Value == check_ref(kind, buf), content


@KINDS
def test_emu_host_offsets(z, kind):
    """Update(data, off, count) for every off in 0..15: slices that start anywhere in a 16-byte word and end anywhere"""
    raw = fill("random", TILE + 200, seed=7).tobytes()
    for off in range(16):
        for count in (0, 1, 3, 15, 16, 17, 127, 128, 129, 4099, TILE - 1, TILE, TILE + 129):
            c = _new(z, kind)
            c.Update(raw, off, count)
            assert c.Value == check_ref(kind, raw[off:off + count]), (off, count)


@KINDS
def test_emu_host_running_updates(z, kind):
    """two Updates split at every chunk and tile edge (the second starts from a running value), and one run of many
    pieces whose ends sit one byte either side of chunk edges"""
    n = 2 * TILE + 129
    for content in FILLS:
        buf = fill(content, n, seed=3)
        want = check_ref(kind, buf)
        for cut in (1, 127, 128, 129, 255, 256, 257, TILE - 129, TILE - 1, TILE, TILE + 1, TILE + 128, 2 * TILE - 1, 2 * TILE,
                    2 * TILE + 1, 2 * TILE + 128, n - 1):
            c = _new(z, kind)
            c.Update(buf, 0, cut)
            assert c.Value == check_ref(kind, buf[:cut]), (content, cut)
            c.Update(buf, cut, n - cut)
            assert c.Value == want, (content, cut)
    buf = fill("random", n, seed=4)
    cuts = sorted({0, n} | {k * CHUNK + d for k in range(1, n // CHUNK, 13) for d in (-1, 0, 1)} | {TILE, 2 * TILE})
    c = _new(z, kind)
    for lo, hi in zip(cuts, cuts[1:]):
        c.Update(buf, lo, hi - lo)
    assert c.Value == check_ref(kind, buf)


@KINDS
def test_emu_host_update_int(z, kind):
    """Update(int) takes the low 8 bits, and mixes with buffer updates"""
    c, want = _new(z, kind), check_ref(kind, b"")
    for v in (0, 255, 0x1FF, -1, 0x80, 7, 0x12345678):
        c.Update(v)
        want = check_ref(kind, bytes([v & 0xFF]), want)
        assert c.Value == want, v
    tail = fill("ff", 300).tobytes()
    c.Update(tail)
    assert c.Value == check_ref(kind, tail, want)


# ---- b200z_checksum_batch_device ----------------------------------------------------------------------------------------
def _side_stream():
    """a stream of its own where there is a device (the CUDA emulator has one stream only)"""
    import torch
    return torch.cuda.Stream() if torch.cuda.is_available() else torch.cuda.current_stream()


def _batch_device(z, kind, blob, offs, lens, seeds, stream=None):
    import torch
    offs = np.ascontiguousarray(offs, dtype=np.int64)
    lens = np.ascontiguousarray(lens, dtype=np.int64)
    v = torch.from_numpy(np.array(seeds, dtype=np.uint32).view(np.int32)).cuda()
    torch.cuda.synchronize()
    s = stream if stream is not None else torch.cuda.current_stream()
    rc = z.lib().b200z_checksum_batch_device(kind, blob.data_ptr(), offs.ctypes.data, lens.ctypes.data, len(lens), v.data_ptr(),
                                             s.cuda_stream)
    assert rc == 0, z.lib().b200z_last_error()
    torch.cuda.synchronize()
    return [int(x) for x in v.cpu().numpy().view(np.uint32)]


@KINDS
def test_emu_batch_device_ragged_streams(z, kind):
    """about 200 streams over one device blob: ragged lengths from the edge list (zero-length ones too), offsets at every
    alignment mod 16, ranges that overlap (the same bytes with different lengths), random seeds, a non-default stream"""
    import torch
    rnd = random.Random(200 + kind)
    host = fill("random", 3 * TILE + 129 + 32, seed=9)
    blob = torch.from_numpy(host).cuda()
    lens = EDGE_LENS[::2] + EDGE_LENS[-24:] + [0, 0, 0]
    offs = [16 * rnd.randrange((host.size - 15 - L) // 16) + i % 16 for i, L in enumerate(lens)]
    for i in range(0, len(lens), 5):  # overlapping: the same start, another length
        L = rnd.choice(EDGE_LENS)
        if offs[i] + L <= host.size:
            offs.append(offs[i])
            lens.append(L)
    assert len(lens) >= 190 and {o % 16 for o in offs} == set(range(16))
    seeds = [_seed(rnd, kind) for _ in lens]
    got = _batch_device(z, kind, blob, offs, lens, seeds, _side_stream())
    want = [check_ref(kind, host[o:o + L], s) for o, L, s in zip(offs, lens, seeds)]
    bad = [(i, offs[i], lens[i]) for i in range(len(lens)) if got[i] != want[i]]
    assert not bad, bad[:10]


def test_emu_batch_device_no_streams(z):
    """n = 0 returns at once and touches nothing"""
    import torch
    v = torch.from_numpy(np.array([0x12345678], dtype=np.uint32).view(np.int32)).cuda()
    for kind in (0, 1):
        assert z.lib().b200z_checksum_batch_device(kind, None, None, None, 0, v.data_ptr(), None) == 0
    assert int(v.cpu().numpy().view(np.uint32)[0]) == 0x12345678


# ---- deflate plans: tiles and multipliers made on the host, several streams per plan ------------------------------------
PAYLOAD_LENS = [0, 1, 129, TILE - 1, TILE, TILE + 1, 2 * TILE + 129]


def _payloads():
    out = []
    for i, n in enumerate(PAYLOAD_LENS):
        if i % 3 == 0:
            out.append(datagen.text_buffer(i, n).tobytes())
        else:
            out.append(fill("ff" if i % 3 == 1 else "random", n, seed=20 + i).tobytes())
    return out


@pytest.mark.parametrize("level", [0, 1, 6])
def test_emu_deflate_plan_checks(z, level):
    """the check values of deflate plans with zlib and raw+CRC framing, and the gzip trailer the deflate pipeline writes"""
    bufs = _payloads()
    outs, checks = z.deflate_batch(bufs, level=level, wrap=WRAP_ZLIB)
    for b, o, c in zip(bufs, outs, checks):
        assert int(c) == check_ref(1, b) and o[-4:] == struct.pack(">I", int(c)), len(b)
        assert zlib.decompress(o) == b
    outs, checks = z.deflate_batch(bufs, level=level, wrap=WRAP_RAW_CRC32)
    for b, o, c in zip(bufs, outs, checks):
        assert int(c) == check_ref(0, b), len(b)
        assert zlib.decompress(o, -15) == b
    p = z.Pipeline.deflate([len(b) for b in bufs], level=level, wrap=WRAP_GZIP)
    ins = [np.frombuffer(b, np.uint8) for b in bufs]
    caps = np.array([z.lib().b200z_deflate_bound(len(b)) + 64 for b in bufs], dtype=np.int64)
    outs = [np.zeros(int(c), np.uint8) for c in caps]
    p.submit(p.pointers([a.ctypes.data if a.size else 0 for a in ins]))
    p.collect(p.pointers([o.ctypes.data for o in outs]), caps)
    p.close()
    for i, b in enumerate(bufs):
        g = outs[i][:int(p.out_len[i])].tobytes()
        assert int(p.check[i]) == check_ref(0, b) and g[:10] == GZIP_HEADER, len(b)
        assert g[-8:] == struct.pack("<II", check_ref(0, b), len(b))
        assert zlib.decompress(g, 31) == b


# ---- inflate plans: tiles over the capacity, multipliers made on the device ---------------------------------------------
def _compress(data, wbits, level=6):
    co = zlib.compressobj(level, zlib.DEFLATED, wbits)
    return co.compress(data) + co.flush()


def _frame(raw, wrap, plain_check, plain_len):
    if wrap == WRAP_ZLIB:
        return b"\x78\x9c" + raw + struct.pack(">I", plain_check)
    if wrap == WRAP_GZIP:
        return GZIP_HEADER + raw + struct.pack("<II", plain_check, plain_len & 0xFFFFFFFF)
    return raw


def _flip_trailer(framed, wrap):
    """one bit of the stored checksum flipped (gzip: the CRC, not ISIZE)"""
    k = len(framed) - (1 if wrap == WRAP_ZLIB else 8)
    return framed[:k] + bytes([framed[k] ^ 0x10]) + framed[k + 1:]


def _inflate(z, comps, caps, wrap, keep=None):
    """one InflatePlan over all streams; returns (outputs, status, in_used, check, stats).  keep: (stream, ranges) -- the
    output of that stream is not copied back whole, only these (lo, hi) ranges plus a SHA-256 of all of it, read back in
    chunks (outputs past 4 GiB)"""
    import torch
    n = len(comps)
    plan = z.InflatePlan([len(c) for c in comps], caps, wrap=wrap)
    h = np.zeros(plan.in_bytes, dtype=np.uint8)
    for i, c in enumerate(comps):
        o = int(plan.data_offsets[i])
        h[o:o + len(c)] = np.frombuffer(c, dtype=np.uint8)
    d_in = torch.from_numpy(h).cuda()
    del h
    d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_ck = torch.zeros(n, dtype=torch.int32, device="cuda")
    t0 = time.time()
    plan.run(d_in, d_out, d_len, d_st, d_ck, d_used)
    torch.cuda.synchronize()
    secs = time.time() - t0
    del d_in
    lens = d_len.cpu().numpy()
    offs = [int(o) for o in plan.out_offsets]
    if keep is None:
        out = d_out.cpu().numpy()
        res = [out[offs[i]:offs[i] + int(lens[i])].tobytes() for i in range(n)]
    else:
        res = []
        for i in range(n):
            o, L = offs[i], int(lens[i])
            parts = {(lo, hi): d_out[o + lo:o + min(hi, L)].cpu().numpy().tobytes() for lo, hi in keep} if i == 0 else {}
            sha = hashlib.sha256()
            for p in range(0, L, 256 * MiB):
                sha.update(d_out[o + p:o + min(p + 256 * MiB, L)].cpu().numpy())
            res.append((L, parts, sha.hexdigest()))
    stats = plan.stats()
    plan.close()
    st, used, ck = d_st.cpu().numpy(), d_used.cpu().numpy(), d_ck.cpu().numpy().view(np.uint32)
    del d_out
    return res, st, used, ck, stats, secs


def _inflate_cases(wrap):
    """every payload at capacities len, len + 1, len + 32768 and 4 len + 65536 (1 MiB as well for the empty one), and
    with its trailer flipped (zlib, gzip)"""
    kind = 1 if wrap == WRAP_ZLIB else 0
    comps, caps, want = [], [], []
    for b in _payloads():
        framed = _frame(_compress(b, -15), wrap, check_ref(kind, b), len(b))
        for cap in [len(b), len(b) + 1, len(b) + TILE, 4 * len(b) + 65536] + ([MiB] if not b else []):
            comps.append(framed)
            caps.append(cap)
            want.append((b, 0))
        if wrap != WRAP_RAW_CRC32:
            comps.append(_flip_trailer(framed, wrap))
            caps.append(len(b) + 1)
            want.append((b, 3 | ((D_ADLER if wrap == WRAP_ZLIB else D_GZIP_CRC) << 8)))
    return comps, caps, want, kind


@pytest.mark.parametrize("wrap", [WRAP_ZLIB, WRAP_GZIP, WRAP_RAW_CRC32], ids=["zlib", "gzip", "raw_crc32"])
@pytest.mark.parametrize("mode", ["parallel", "serial"])
def test_emu_inflate_plan_checks(z, wrap, mode):
    comps, caps, want, kind = _inflate_cases(wrap)
    run = _inflate if mode == "parallel" else (lambda *a: _serial(_inflate, *a))
    res, st, used, ck, stats, _ = run(z, comps, caps, wrap)
    assert stats["parallel"] == (1 if mode == "parallel" else 0)
    for i, (b, status) in enumerate(want):
        assert int(st[i]) == status, (i, len(b), caps[i], hex(int(st[i])))
        assert res[i] == b and int(used[i]) == len(comps[i]), (i, len(b), caps[i])
        assert int(ck[i]) == check_ref(kind, b), (i, len(b), caps[i], hex(int(ck[i])))


# ---- past 4 GiB ---------------------------------------------------------------------------------------------------------
def _host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _need(device_bytes, host_bytes=0):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < device_bytes + GiB // 2:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free" % (device_bytes / GiB, free / GiB))
    avail = _host_available()
    if avail < host_bytes + GiB:
        pytest.skip("needs %.1f GiB of available host memory, %.1f GiB available" % (host_bytes / GiB, avail / GiB))


def _release(z):
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    z.lib().b200z_release_cached()


@pytest.fixture(scope="class")
def big_blob(z):
    """2^32 + 64 KiB random bytes on the device"""
    import torch
    _need(BIG + 64 * 1024 + GiB)
    g = torch.Generator(device="cuda")
    g.manual_seed(0x4A11)
    blob = torch.empty(BIG + 64 * 1024, dtype=torch.uint8, device="cuda").random_(0, 256, generator=g)
    yield blob
    del blob
    _release(z)


class TestBlobPast4GiB:
    @KINDS
    def test_batch_device(self, z, big_blob, kind):
        """offset 0 with lengths 2^32 - 1, 2^32, 2^32 + 1 and 2^32 + 32768 + 129 (one seed), offset 13 with 2^32 + 7"""
        rnd = random.Random(41 + kind)
        seed_a, seed_b = _seed(rnd, kind), _seed(rnd, kind)
        lens = [BIG - 1, BIG, BIG + 1, BIG + TILE + 129, BIG + 7]
        offs = [0, 0, 0, 0, 13]
        got = _batch_device(z, kind, big_blob, offs, lens, [seed_a] * 4 + [seed_b], _side_stream())
        want, v, pos = [], seed_a, 0
        for L in lens[:4]:  # the four prefixes of one range: one running value
            v = check_ref(kind, big_blob, v, pos, L)
            pos = L
            want.append(v)
        want.append(check_ref(kind, big_blob, seed_b, 13, 13 + lens[4]))
        assert got == want, [(L, hex(g), hex(w)) for L, g, w in zip(lens, got, want)]

    @KINDS
    def test_host_update(self, z, big_blob, kind):
        """Crc32 / Adler32.Update on a host buffer of 2^32 + 40003 bytes: whole, and as two Updates split below 4 GiB"""
        n = BIG + 40003
        _need(n + 256 * MiB, n)
        host = big_blob[:n].cpu().numpy()
        want = check_ref(kind, host)
        c = _new(z, kind)
        c.Update(host)
        whole = c.Value
        cut = 3 * GiB + 12345
        c = _new(z, kind)
        c.Update(host, 0, cut)
        c.Update(host, cut, n - cut)
        del host
        _release(z)
        assert (hex(whole), hex(c.Value)) == (hex(want), hex(want))


BIG_OUT = BIG + 3 * MiB + 12345


@pytest.fixture(scope="module")
def big_stream():
    """a raw DEFLATE stream whose output is BIG_OUT bytes, made of pieces that each end in Z_FULL_FLUSH (independent, so
    one compressed piece can be repeated): a shared piece of log text between small unique pieces (a counter and random
    bytes: the 32 KiB tile at 2^32 + 32768 k never holds the same bytes as tile k), and an empty final block.
    Returns (raw, plain pieces in order, CRC-32, Adler-32, SHA-256 of the output)."""
    shared = datagen.log_stream(61 * MiB + 4093).tobytes()
    reps = BIG_OUT // len(shared)
    q, r = divmod(BIG_OUT - reps * len(shared), reps)
    rng = datagen.Rng(0x4617)

    def piece(b):
        co = zlib.compressobj(6, zlib.DEFLATED, -15)
        return co.compress(b) + co.flush(zlib.Z_FULL_FLUSH)
    c_shared = piece(shared)
    plain, comp = [], []
    for k in range(reps):
        u = k.to_bytes(8, "little") + rng.bytes(q + (k < r) - 8).tobytes()
        plain += [shared, u]
        comp += [c_shared, piece(u)]
    comp.append(zlib.compressobj(6, zlib.DEFLATED, -15).flush())  # the final block: empty
    assert sum(len(p) for p in plain) == BIG_OUT
    crc, adler, sha = 0, 1, hashlib.sha256()
    for p in plain:
        crc, adler = zlib.crc32(p, crc), zlib.adler32(p, adler)
        sha.update(p)
    return b"".join(comp), plain, crc, adler, sha.hexdigest()


def _plain_range(plain, lo, hi):
    out, pos = [], 0
    for p in plain:
        a, b = max(lo, pos), min(hi, pos + len(p))
        if a < b:
            out.append(p[a - pos:b - pos])
        pos += len(p)
    return b"".join(out)


WINDOWS = [(0, MiB), (BIG - MiB, BIG + MiB), (BIG_OUT - MiB, BIG_OUT)]


def _check_big(res, st, used, ck, framed, want_status, want_check, stream_info):
    raw, plain, _, _, sha = stream_info
    L, parts, got_sha = res[0]
    assert (int(st[0]), L, int(used[0])) == (0, BIG_OUT, len(framed))
    assert hex(int(ck[0])) == hex(want_check)
    for lo, hi in WINDOWS:
        assert parts[(lo, hi)] == _plain_range(plain, lo, hi), (lo, hi)
    assert got_sha == sha
    if len(res) > 1:
        assert int(st[1]) == want_status and hex(int(ck[1])) == hex(want_check)


@pytest.mark.parametrize("wrap", [WRAP_GZIP, WRAP_ZLIB, WRAP_RAW_CRC32], ids=["gzip", "zlib", "raw_crc32"])
def test_inflate_past_4gib(z, big_stream, wrap):
    """one stream whose output is just over 4 GiB, and the same with its trailer flipped, in one plan of the serial kernel
    (the block-parallel pipeline hands such a stream to it; test_inflate_past_4gib_handed_back runs that path)"""
    raw, plain, crc, adler, _ = big_stream
    kind_check = adler if wrap == WRAP_ZLIB else crc
    framed = _frame(raw, wrap, kind_check, BIG_OUT)
    comps = [framed] if wrap == WRAP_RAW_CRC32 else [framed, _flip_trailer(framed, wrap)]
    _need(len(comps) * (BIG_OUT + len(framed)) + GiB, 2 * len(framed))
    res, st, used, ck, stats, secs = _serial(_inflate, z, comps, [BIG_OUT] * len(comps), wrap, WINDOWS)
    print("serial kernel: %d stream(s) of %d bytes from %d in %.1f s" % (len(comps), BIG_OUT, len(framed), secs))
    del comps
    _release(z)
    assert stats["parallel"] == 0
    _check_big(res, st, used, ck, framed, 3 | ((D_ADLER if wrap == WRAP_ZLIB else D_GZIP_CRC) << 8), kind_check, big_stream)


def test_inflate_past_4gib_handed_back(z, big_stream):
    """the gzip member through the default plan: the block-parallel pipeline hands the stream to the serial kernel
    (its pools for a 4 GiB output take about 12 GiB of their own)"""
    raw, plain, crc, _, _ = big_stream
    framed = _frame(raw, WRAP_GZIP, crc, BIG_OUT)
    _need(BIG_OUT + len(framed) + BIG_OUT // 3 * 8 + 2 * GiB, 2 * len(framed))
    res, st, used, ck, stats, secs = _inflate(z, [framed], [BIG_OUT], WRAP_GZIP, WINDOWS)
    print("default plan: %d bytes from %d in %.1f s, %s" % (BIG_OUT, len(framed), secs, stats))
    _release(z)
    assert stats["parallel"] == 1 and stats["handed_back"] == 1, stats
    _check_big(res, st, used, ck, framed, 0, crc, big_stream)


def test_gzip_output_stream_one_write_past_4gib(z):
    """one GZipOutputStream.Write of about 4.2 GiB at the default level: the CRC-32 trailer comes from one Crc32.Update
    over the whole buffer; a sink that inflates as the bytes arrive must reach the end with no "incorrect data check".
    (The handle's SetInput takes an int32 count, as Deflater.SetInput does: Write feeds longer spans in pieces, and a
    SetInput of more than 2^31 - 1 bytes is refused instead of being cut to the low 32 bits of its length.)"""
    n = BIG + 200 * MiB + 777
    _need(n + 2 * GiB, 2 * n)
    with pytest.raises(ValueError):
        z.Deflater().SetInput(np.zeros(1 << 31, np.uint8))
    shared = datagen.log_stream(61 * MiB + 4093)
    host = np.resize(shared, n)  # period 61 MiB + 4093: the bytes at 2^32 + x are not the bytes at x
    host[BIG - 3:BIG + 5] = np.frombuffer(b"4GiBedge", np.uint8)
    want = check_ref(0, host)

    class Sink:
        def __init__(self):
            self.d = zlib.decompressobj(31)
            self.crc, self.n, self.tail = 0, 0, b""

        def write(self, b):
            out = self.d.decompress(b)
            self.crc = zlib.crc32(out, self.crc)
            self.n += len(out)
            self.tail = (self.tail + bytes(b))[-8:]

    sink = Sink()
    g = z.GZipOutputStream(sink)
    g.ModifiedTime = 0
    t0 = time.time()
    g.Write(host)
    g.Finish()
    print("GZipOutputStream: one Write of %d bytes in %.1f s" % (n, time.time() - t0))
    del host, g
    _release(z)
    sink.d.flush()
    assert sink.d.eof and sink.n == n and sink.crc == want
    assert sink.tail == struct.pack("<II", want, n & 0xFFFFFFFF)
