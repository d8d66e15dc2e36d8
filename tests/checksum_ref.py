"""Plain references for CRC-32 and Adler-32, to hold the tile-parallel checksum kernel (b200z_checksum.cu) against.

crc32_bitwise / adler32_def restate the two checksums from their definitions, with no tables and no deferred reductions:
slow, but nothing in them can share a mistake with the kernel's combination identities (b200z_crc.cuh).  The CPU tier ties
them to zlib and to the oracle on small inputs; crc32_ref / adler32_ref are zlib over bounded chunks with a running value,
for inputs too long for the definitions (up to and past 4 GiB, from host memory or from a device tensor copied back a chunk
at a time so that no second full-size host copy is made)."""
import zlib

import numpy as np

CRC_POLY = 0xEDB88320  # reflected x^32 + x^26 + x^23 + x^22 + x^16 + x^12 + x^11 + x^10 + x^8 + x^7 + x^5 + x^4 + x^2 + x + 1
ADLER_BASE = 65521
CHUNK = 256 << 20


def crc32_bitwise(data, seed=0):
    """CRC-32/ISO-HDLC one bit at a time.  `seed` is any 32-bit running value (Crc32.Value after earlier updates): the
    register starts as seed ^ 0xFFFFFFFF and the result is the register ^ 0xFFFFFFFF."""
    reg = (seed & 0xFFFFFFFF) ^ 0xFFFFFFFF
    for b in bytes(data):
        reg ^= b
        for _ in range(8):
            reg = (reg >> 1) ^ CRC_POLY if reg & 1 else reg >> 1
    return reg ^ 0xFFFFFFFF


def adler32_def(data, seed=1):
    """Adler-32 from its definition with Python integers.  With n bytes b_0..b_{n-1} and the seed's halves s1 (low), s2
    (high): s1' = s1 + sum b_i, s2' = s2 + n * s1 + sum (n - i) * b_i, each reduced mod 65521 once, at the end.  The seed
    is a valid Adler value (both halves below 65521)."""
    s1, s2 = seed & 0xFFFF, seed >> 16
    assert s1 < ADLER_BASE and s2 < ADLER_BASE, hex(seed)
    d = bytes(data)
    n = len(d)
    a = s1 + sum(d)
    b = s2 + n * s1 + sum((n - i) * x for i, x in enumerate(d))
    return ((b % ADLER_BASE) << 16) | (a % ADLER_BASE)


def _chunks(data, lo=0, hi=None):
    """host bytes / numpy array / torch tensor (any device) -> numpy uint8 pieces of at most CHUNK bytes"""
    if hasattr(data, "is_cuda"):  # a torch tensor: one chunk at a time back to the host
        hi = data.numel() if hi is None else hi
        for p in range(lo, hi, CHUNK):
            yield data[p:min(p + CHUNK, hi)].cpu().numpy()
        return
    a = data if isinstance(data, np.ndarray) else np.frombuffer(data, dtype=np.uint8)
    hi = a.size if hi is None else hi
    for p in range(lo, hi, CHUNK):
        yield a[p:min(p + CHUNK, hi)]


def crc32_ref(data, seed=0, lo=0, hi=None):
    """zlib's CRC-32 of data[lo:hi] from the running value `seed`"""
    v = seed
    for c in _chunks(data, lo, hi):
        v = zlib.crc32(c, v)
    return v


def adler32_ref(data, seed=1, lo=0, hi=None):
    """zlib's Adler-32 of data[lo:hi] from the running value `seed`"""
    v = seed
    for c in _chunks(data, lo, hi):
        v = zlib.adler32(c, v)
    return v


def check_ref(kind, data, seed=None, lo=0, hi=None):
    """kind 0: CRC-32 (Reset value 0), kind 1: Adler-32 (Reset value 1)"""
    if kind == 0:
        return crc32_ref(data, 0 if seed is None else seed, lo, hi)
    return adler32_ref(data, 1 if seed is None else seed, lo, hi)
