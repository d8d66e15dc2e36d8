"""CPU tier: the CRC-32/BZIP2 references (tests/bzip2crc_ref.py) against the reference's known answers and each other, the
BZip2Crc mirror's Value before any update, and the small cases of tests/test_gpu_bzip2crc.py ("emu") on the CUDA emulator in
the default schedule and with the threads and blocks resumed in reverse order."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import bzip2crc_ref
from bzip2crc_ref import BZIP2_POLY, bzip2crc_bitwise, check_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = b"123456789"  # ChecksumTests.cs:14
LONG_CHECK = CHECK * 4  # ChecksumTests.cs:17-22


def _inputs():
    rnd = np.random.default_rng(11)
    for n in range(301):
        yield "zeros", bytes(n)
        yield "ff", b"\xff" * n
        yield "random", rnd.integers(0, 256, n, dtype=np.uint8).tobytes()


@pytest.mark.parametrize("ref", ["bitwise", "oracle"])
def test_known_answers(ref):
    """ChecksumTests.cs:67-105: "123456789", longCheck, the ArraySegment "456" (offset 3) and "789123456789123456"
    (offset 15, 18 bytes)"""
    f = bzip2crc_bitwise if ref == "bitwise" else bzip2crc_ref.oracle
    assert f(CHECK) == 0xFC891918
    assert f(LONG_CHECK) == 0xEE53D2B2
    assert f(CHECK[3:6]) == 0x001D0511
    assert f(LONG_CHECK[15:33]) == 0x025846E0


def test_value_after_construction_and_reset():
    """Value is ~checkValue and Reset sets checkValue to 0xFFFFFFFF, so Value is 0 before any update and after Reset"""
    import sharpziplib_b200 as z
    assert bzip2crc_ref.oracle_reset_value() == 0
    c = z.BZip2Crc()
    assert c.Value == c.value == 0
    c._value = 0x12345678  # as if updated: Reset needs no device
    c.Reset()
    assert c.Value == 0


def test_definition_matches_the_oracle_from_running_values():
    """every length 0-300 in three contents, from Reset and from random running values (0xFFFFFFFF included)"""
    rnd = random.Random(12)
    for i, (name, d) in enumerate(_inputs()):
        assert bzip2crc_bitwise(d) == bzip2crc_ref.oracle(d), (name, len(d))
        seed = rnd.getrandbits(32) if i % 7 else 0xFFFFFFFF
        assert bzip2crc_bitwise(d, seed) == bzip2crc_ref.oracle(d, seed), (name, len(d), hex(seed))


def test_update_int_takes_the_low_byte():
    rnd = random.Random(13)
    v = 0
    for b in (0, 255, 256, 0x1FF, -1, -256, 0x12345678) + tuple(rnd.randrange(-2 ** 31, 2 ** 31) for _ in range(50)):
        nxt = bzip2crc_ref.oracle_update_int(v, b)
        assert nxt == bzip2crc_bitwise(bytes([b & 0xFF]), v) == bzip2crc_ref.oracle(bytes([b & 0xFF]), v), b
        v = nxt


def _mulmod(a, b):
    """a(x) * b(x) mod P, normal bit order (x^0 = bit 0)"""
    p = 0
    for i in range(32):
        if a >> i & 1:
            p ^= b
        b = ((b << 1) ^ BZIP2_POLY) & 0xFFFFFFFF if b & 0x80000000 else b << 1
    return p


def _xpow8(n):
    p, sq = 1, 1 << 8
    while n:
        if n & 1:
            p = _mulmod(sq, p)
        sq = _mulmod(sq, sq)
        n >>= 1
    return p


def _raw(reg, data):
    """the register after feeding data from register `reg`, no final xor"""
    return bzip2crc_bitwise(data, reg ^ 0xFFFFFFFF) ^ 0xFFFFFFFF


def test_combination_identity():
    """raw(0, A || B) = raw(0, A) * x^(8 |B|) xor raw(0, B) and raw(s, D) = s * x^(8 |D|) xor raw(0, D), in the normal bit
    order the kernel combines its chunk and tile partials with; and Value from v0 = raw(~v0, M) ^ ~0"""
    rnd = np.random.default_rng(14)
    d = rnd.integers(0, 256, 700, dtype=np.uint8).tobytes()
    for cut in (0, 1, 3, 4, 5, 127, 128, 129, 300, 699, 700):
        a, b = d[:cut], d[cut:]
        assert _raw(0, d) == _mulmod(_raw(0, a), _xpow8(len(b))) ^ _raw(0, b), cut
    for s in (1, 0x80000000, 0xFFFFFFFF, 0x1234ABCD):
        for n in (0, 1, 17, 128, 513):
            assert _raw(s, d[:n]) == _mulmod(s, _xpow8(n)) ^ _raw(0, d[:n]), (hex(s), n)
    v0 = 0xCAFEF00D
    assert bzip2crc_bitwise(d, v0) == (_mulmod(v0 ^ 0xFFFFFFFF, _xpow8(len(d))) ^ _raw(0, d)) ^ 0xFFFFFFFF
    assert _xpow8(0) == 1 and _xpow8(4) == BZIP2_POLY  # x^32 mod P is P without its x^32 term


def test_chunked_reference_over_chunk_edges(monkeypatch):
    """the chunked reference (what the GPU tier uses for long inputs) gives the whole-buffer value, with a seed and for a
    sub-range"""
    import checksum_ref
    monkeypatch.setattr(checksum_ref, "CHUNK", 1000)
    d = np.random.default_rng(15).integers(0, 256, 10007, dtype=np.uint8)
    b = d.tobytes()
    for seed in (None, 0x12345678):
        assert check_ref(2, d, seed) == bzip2crc_ref.oracle(b, seed or 0)
    assert check_ref(2, d, None, 999, 5003) == bzip2crc_ref.oracle(b[999:5003])
    assert check_ref(2, d, 77, 13, 10007) == bzip2crc_ref.oracle(b[13:], 77)
    assert check_ref(0, d) == checksum_ref.check_ref(0, d) and check_ref(1, d, 5) == checksum_ref.check_ref(1, d, 5)


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_bzip2crc_kernel_on_the_emulator(order):
    env = dict(os.environ)
    if order == "rev":
        env["B200Z_EMU_ORDER"] = "rev"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"),
                        os.path.join(ROOT, "tests", "test_gpu_bzip2crc.py"), "-k", "emu"],
                       capture_output=True, text=True, timeout=1500, env=env)
    assert r.returncode == 0 and " passed" in r.stdout and "deselected" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
