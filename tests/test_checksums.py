"""CPU tier: the plain checksum references (tests/checksum_ref.py) agree with zlib and with the oracle on small inputs, and
the checksum kernel runs the GPU tier's small cases (tests/test_gpu_checksums.py, "emu") on the CUDA emulator, in the
default schedule and with the threads and blocks resumed in reverse order."""
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest

from checksum_ref import adler32_def, check_ref, crc32_bitwise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs():
    rnd = np.random.default_rng(5)
    for n in range(301):
        yield "zeros", bytes(n)
        yield "ff", b"\xff" * n
        yield "random", rnd.integers(0, 256, n, dtype=np.uint8).tobytes()


def test_definitions_match_zlib_and_the_oracle(oracle):
    for name, d in _inputs():
        assert crc32_bitwise(d) == zlib.crc32(d) == oracle.crc32(d), (name, len(d))
        assert adler32_def(d) == zlib.adler32(d) == oracle.adler32(d), (name, len(d))


def test_definitions_from_running_values(oracle):
    """any 32-bit CRC seed; Adler seeds with both halves below 65521, the largest included"""
    rnd = random.Random(6)
    adler_seeds = [1, 0, 0xFFF0FFF0, 0xFFF00000, 0x0000FFF0]
    for i, (name, d) in enumerate(_inputs()):
        cs = rnd.getrandbits(32) if i % 7 else 0xFFFFFFFF
        a_s = adler_seeds[i] if i < len(adler_seeds) else (rnd.randrange(65521) << 16) | rnd.randrange(65521)
        assert crc32_bitwise(d, cs) == zlib.crc32(d, cs) == oracle.crc32_update(cs, d), (name, len(d), cs)
        assert adler32_def(d, a_s) == zlib.adler32(d, a_s) == oracle.adler32_update(a_s, d), (name, len(d), a_s)


def test_chunked_references_over_chunk_edges(monkeypatch):
    """the zlib references over pieces (what the GPU tier uses for long inputs) give the whole-buffer value, with a seed and
    for a sub-range"""
    import checksum_ref
    monkeypatch.setattr(checksum_ref, "CHUNK", 1000)
    d = np.random.default_rng(7).integers(0, 256, 10007, dtype=np.uint8)
    b = d.tobytes()
    for seed in (None, 0x12345678):
        assert check_ref(0, d, seed) == zlib.crc32(b, seed or 0)
        assert check_ref(1, b, seed) == zlib.adler32(b, seed or 1)
    assert check_ref(0, d, None, 999, 5003) == zlib.crc32(b[999:5003])
    assert check_ref(1, d, 77, 13, 10007) == zlib.adler32(b[13:], 77)


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_checksum_kernel_on_the_emulator(order):
    env = dict(os.environ)
    if order == "rev":
        env["B200Z_EMU_ORDER"] = "rev"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"),
                        os.path.join(ROOT, "tests", "test_gpu_checksums.py"), "-k", "emu"],
                       capture_output=True, text=True, timeout=1500, env=env)
    assert r.returncode == 0 and " passed" in r.stdout and "deselected" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
