"""GPU tier: CRC-32/BZIP2, kind 2 of the checksum kernel (b200z_checksum.cu), against the bitwise definition and the
BZip2Crc restatement (tests/bzip2crc_ref.py) at the edges tests/test_gpu_checksums.py covers for the other two kinds: every
length up to two chunks, every chunk and tile edge of the first three tiles, all-0xFF and period-128 contents, running
values as seeds, streams past 4 GiB, and the reference benchmark's 256 MiB input.

Both entry points are covered: BZip2Crc (host buffers, b200z_bzip2crc) and b200z_checksum_batch_device(kind = 2).  Tests
whose name holds "emu" are small enough for the CUDA emulator; the CPU tier runs them there.  The cases past 4 GiB check
free device and host memory first and skip, saying why, when it is short."""
import random

import numpy as np
import pytest

import bzip2crc_ref
from bzip2crc_ref import bzip2crc_bitwise, check_ref
from test_gpu_checksums import (BIG, CHUNK, EDGE_LENS, FILLS, GiB, MiB, TILE, _batch_device, _need, _release, _side_stream,
                                big_blob, fill)  # noqa: F401 (big_blob: the 4 GiB device blob fixture, for TestBlobPast4GiB)

pytestmark = pytest.mark.gpu

B200Z_E_ARG = 1
CHECK = b"123456789"  # ChecksumTests.cs:14, `check`
LONG_CHECK = CHECK * 4  # ChecksumTests.cs:17-22, `longCheck`
RANDOM_1_LEN = 256 * MiB  # benchmark/.../Checksum/BZip2Crc.cs: ChunkCount * ChunkSize of new Random(1).NextBytes


# ---- BZip2Crc on host buffers -------------------------------------------------------------------------------------------
def test_emu_known_answers(z):
    """the reference's four known answers (ChecksumTests.cs:67-105), through Update(bytes) and Update(ArraySegment)"""
    c = z.BZip2Crc()
    assert c.Value == 0
    c.Update(CHECK)
    assert c.Value == 0xFC891918
    c.Reset()
    assert c.Value == 0
    c.Update(LONG_CHECK)
    assert c.Value == 0xEE53D2B2
    c = z.BZip2Crc()
    c.Update(CHECK, 3, 3)
    assert c.Value == 0x001D0511
    c = z.BZip2Crc()
    c.Update(LONG_CHECK, 15, 18)
    assert c.Value == 0x025846E0


@pytest.mark.parametrize("content", FILLS)
def test_emu_host_every_edge_length(z, content):
    """every length 0-260 and 32768 k + {-129, -128, -1, 0, 1, 127, 128, 129}, k = 1..3"""
    buf = fill(content, EDGE_LENS[-1])
    for n in EDGE_LENS:
        c = z.BZip2Crc()
        c.Update(buf[:n])
        want = bzip2crc_bitwise(buf[:n]) if n <= 2 * CHUNK else bzip2crc_ref.oracle(buf[:n])
        assert c.Value == want, (content, n, hex(c.Value))


@pytest.mark.parametrize("content", FILLS)
def test_host_five_mib(z, content):
    n = (5 << 20) + 7
    buf = fill(content, n)
    c = z.BZip2Crc()
    c.Update(buf)
    assert c.Value == check_ref(2, buf), content


def test_emu_host_offsets(z):
    """Update(data, off, count) for every off in 0..15: slices that start anywhere in a 16-byte word and end anywhere"""
    raw = fill("random", TILE + 200, seed=7).tobytes()
    for off in range(16):
        for count in (0, 1, 3, 15, 16, 17, 127, 128, 129, 4099, TILE - 1, TILE, TILE + 129):
            c = z.BZip2Crc()
            c.Update(raw, off, count)
            assert c.Value == check_ref(2, raw[off:off + count]), (off, count)


def test_emu_host_running_updates(z):
    """two Updates split at every chunk and tile edge (the second starts from a running value), and one run of many
    pieces whose ends sit one byte either side of chunk edges"""
    n = 2 * TILE + 129
    for content in FILLS:
        buf = fill(content, n, seed=3)
        want = check_ref(2, buf)
        for cut in (1, 127, 128, 129, 255, 256, 257, TILE - 129, TILE - 1, TILE, TILE + 1, TILE + 128, 2 * TILE - 1, 2 * TILE,
                    2 * TILE + 1, 2 * TILE + 128, n - 1):
            c = z.BZip2Crc()
            c.Update(buf, 0, cut)
            assert c.Value == check_ref(2, buf[:cut]), (content, cut)
            c.Update(buf, cut, n - cut)
            assert c.Value == want, (content, cut)
    buf = fill("random", n, seed=4)
    cuts = sorted({0, n} | {k * CHUNK + d for k in range(1, n // CHUNK, 13) for d in (-1, 0, 1)} | {TILE, 2 * TILE})
    c = z.BZip2Crc()
    for lo, hi in zip(cuts, cuts[1:]):
        c.Update(buf, lo, hi - lo)
    assert c.Value == check_ref(2, buf)


def test_emu_host_update_int(z):
    """Update(int) takes the low 8 bits (values above 255 and negative ones too), and mixes with buffer updates"""
    c, want = z.BZip2Crc(), 0
    for v in (0, 255, 0x1FF, -1, 0x80, 7, 0x12345678, 256, -256):
        c.Update(v)
        nxt = bzip2crc_ref.oracle_update_int(want, v)
        assert nxt == bzip2crc_bitwise(bytes([v & 0xFF]), want), v
        want = nxt
        assert c.Value == want, v
    tail = fill("ff", 300).tobytes()
    c.Update(tail)
    assert c.Value == check_ref(2, tail, want)


# ---- b200z_checksum_batch_device(kind = 2) ------------------------------------------------------------------------------
def test_emu_batch_device_ragged_streams(z):
    """about 200 streams over one device blob: ragged lengths from the edge list (zero-length ones too), offsets at every
    alignment mod 16, ranges that overlap (the same bytes with different lengths), random seeds, a non-default stream"""
    import torch
    rnd = random.Random(202)
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
    seeds = [rnd.getrandbits(32) for _ in lens]
    got = _batch_device(z, 2, blob, offs, lens, seeds, _side_stream())
    want = [check_ref(2, host[o:o + L], s) for o, L, s in zip(offs, lens, seeds)]
    bad = [(i, offs[i], lens[i]) for i in range(len(lens)) if got[i] != want[i]]
    assert not bad, bad[:10]


def test_emu_batch_device_three_kinds_one_blob(z):
    """the same streams over one blob run as kind 0, 1 and 2 in turn: each result is its own kind's checksum"""
    import torch
    rnd = random.Random(203)
    host = fill("random", 2 * TILE + 300, seed=10)
    blob = torch.from_numpy(host).cuda()
    lens = [0, 1, 5, 128, 129, TILE - 1, TILE, TILE + 1, 2 * TILE + 129]
    offs = [rnd.randrange(host.size - L + 1) for L in lens]
    for kind in (0, 1, 2):
        got = _batch_device(z, kind, blob, offs, lens, [check_ref(kind, b"")] * len(lens))
        assert got == [check_ref(kind, host[o:o + L]) for o, L in zip(offs, lens)], kind


def test_emu_batch_device_no_streams_and_bad_kinds(z):
    """n = 0 returns at once and touches nothing; kinds outside 0..2 are refused before anything runs"""
    import torch
    v = torch.from_numpy(np.array([0x12345678], dtype=np.uint32).view(np.int32)).cuda()
    blob = torch.zeros(64, dtype=torch.uint8).cuda()
    offs, lens = np.zeros(1, np.int64), np.full(1, 64, np.int64)
    assert z.lib().b200z_checksum_batch_device(2, None, None, None, 0, v.data_ptr(), None) == 0
    for kind in (3, -1):
        assert z.lib().b200z_checksum_batch_device(kind, blob.data_ptr(), offs.ctypes.data, lens.ctypes.data, 1, v.data_ptr(),
                                                   None) == B200Z_E_ARG, kind
    assert int(v.cpu().numpy().view(np.uint32)[0]) == 0x12345678


# ---- past 4 GiB ---------------------------------------------------------------------------------------------------------
class TestBlobPast4GiB:
    def test_batch_device(self, z, big_blob):
        """offset 0 with lengths 2^32 - 1, 2^32, 2^32 + 1 and 2^32 + 32768 + 129 (one seed), offset 13 with 2^32 + 7"""
        rnd = random.Random(43)
        seed_a, seed_b = rnd.getrandbits(32), rnd.getrandbits(32)
        lens = [BIG - 1, BIG, BIG + 1, BIG + TILE + 129, BIG + 7]
        offs = [0, 0, 0, 0, 13]
        got = _batch_device(z, 2, big_blob, offs, lens, [seed_a] * 4 + [seed_b], _side_stream())
        want, v, pos = [], seed_a, 0
        for L in lens[:4]:  # the four prefixes of one range: one running value
            v = check_ref(2, big_blob, v, pos, L)
            pos = L
            want.append(v)
        want.append(check_ref(2, big_blob, seed_b, 13, 13 + lens[4]))
        assert got == want, [(L, hex(g), hex(w)) for L, g, w in zip(lens, got, want)]

    def test_host_update(self, z, big_blob):
        """BZip2Crc.Update on a host buffer of 2^32 + 40003 bytes: whole, and as two Updates split below 4 GiB"""
        n = BIG + 40003
        _need(n + 256 * MiB, n)
        host = big_blob[:n].cpu().numpy()
        want = check_ref(2, host)
        c = z.BZip2Crc()
        c.Update(host)
        whole = c.Value
        cut = 3 * GiB + 12345
        c = z.BZip2Crc()
        c.Update(host, 0, cut)
        c.Update(host, cut, n - cut)
        del host
        _release(z)
        assert (hex(whole), hex(c.Value)) == (hex(want), hex(want))


# ---- the reference benchmark's input ------------------------------------------------------------------------------------
def test_reference_benchmark_input(z, oracle):
    """256 MiB of new Random(1).NextBytes: one Update, and 256 Updates of 1 MiB, both equal to the restatement"""
    data = oracle.dotnet_random_bytes(1, RANDOM_1_LEN)
    want = bzip2crc_ref.oracle(data)
    c = z.BZip2Crc()
    c.Update(data)
    assert c.Value == want
    c = z.BZip2Crc()
    for k in range(256):
        c.Update(data, k * MiB, MiB)
    assert c.Value == want
