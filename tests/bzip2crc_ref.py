"""TEST INFRASTRUCTURE: references for CRC-32/BZIP2 (BZip2Crc), to hold kind 2 of the checksum kernel (b200z_checksum.cu)
against.

bzip2crc_bitwise restates the checksum from its definition, one bit at a time with no tables: slow, but it cannot share a
mistake with the kernel's tables or combination identities.  oracle() is BZip2Crc restated over its slicing-by-16 tables
(tests/cpu_model/bzip2crc_model.cpp, built on first use into tests/cpu_model/_build); bzip2crc_ref runs it over bounded
chunks with a running value, for inputs up to and past 4 GiB, from host memory or from a device tensor copied back a chunk
at a time.  check_ref extends checksum_ref.check_ref with kind 2."""
import ctypes as C
import os
import subprocess

import numpy as np

import checksum_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_model", "bzip2crc_model.cpp")
_SO = os.path.join(ROOT, "tests", "cpu_model", "_build", "libbzip2crc_model.so")
_L = None

BZIP2_POLY = 0x04C11DB7  # x^32 + x^26 + x^23 + x^22 + x^16 + x^12 + x^11 + x^10 + x^8 + x^7 + x^5 + x^4 + x^2 + x + 1, normal


def lib():
    global _L
    if _L is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = _SO + ".%d" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", tmp, _SRC])
            os.replace(tmp, _SO)
        L = C.CDLL(_SO)
        L.bz2crc_model_update.restype = C.c_uint32
        L.bz2crc_model_update.argtypes = [C.c_uint32, C.c_void_p, C.c_uint64]
        L.bz2crc_model_update_int.restype = C.c_uint32
        L.bz2crc_model_update_int.argtypes = [C.c_uint32, C.c_int32]
        L.bz2crc_model_reset_value.restype = C.c_uint32
        L.bz2crc_model_reset_value.argtypes = []
        _L = L
    return _L


def bzip2crc_bitwise(data, seed=0):
    """CRC-32/BZIP2 one bit at a time.  `seed` is any 32-bit running value (BZip2Crc.Value after earlier updates): the
    register starts as seed ^ 0xFFFFFFFF, each byte enters at the top, most significant bit first, and the result is the
    register ^ 0xFFFFFFFF."""
    reg = (seed & 0xFFFFFFFF) ^ 0xFFFFFFFF
    for b in bytes(data):
        reg ^= b << 24
        for _ in range(8):
            reg = ((reg << 1) ^ BZIP2_POLY) & 0xFFFFFFFF if reg & 0x80000000 else (reg << 1) & 0xFFFFFFFF
    return reg ^ 0xFFFFFFFF


def oracle(data, seed=0):
    """the BZip2Crc restatement: Value after Update(data) from the running value `seed`"""
    a = data if isinstance(data, np.ndarray) else np.frombuffer(bytes(data), dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return lib().bz2crc_model_update(seed & 0xFFFFFFFF, a.ctypes.data if a.size else None, a.size)


def oracle_update_int(seed, bval):
    """the BZip2Crc restatement: Value after Update(int bval) from the running value `seed`"""
    return lib().bz2crc_model_update_int(seed & 0xFFFFFFFF, bval)


def oracle_reset_value():
    return lib().bz2crc_model_reset_value()


def bzip2crc_ref(data, seed=0, lo=0, hi=None):
    """the restatement over data[lo:hi] from the running value `seed`, one chunk of checksum_ref.CHUNK bytes at a time"""
    v = seed
    for c in checksum_ref._chunks(data, lo, hi):
        v = oracle(c, v)
    return v


def check_ref(kind, data, seed=None, lo=0, hi=None):
    """kind 0: CRC-32 (Reset value 0), kind 1: Adler-32 (Reset value 1), kind 2: CRC-32/BZIP2 (Reset value 0)"""
    if kind == 2:
        return bzip2crc_ref(data, 0 if seed is None else seed, lo, hi)
    return checksum_ref.check_ref(kind, data, seed, lo, hi)
