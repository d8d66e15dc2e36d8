"""TEST INFRASTRUCTURE: the LZW (.Z) reference of tests/cpu_model/lzw_model.cpp -- LzwInputStream restated with its 8 KiB
buffer over a base stream with a chosen Read() schedule, and a compress(1)-format encoder.  Builds the library on first use
into tests/cpu_model/_build."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpu_model", "lzw_model.cpp")
_SO = os.path.join(ROOT, "tests", "cpu_model", "_build", "liblzw_model.so")
_L = None

# (kind, a, b) -> the reference's exception message; kind 6 is a non-SharpZip exception
MESSAGES = {
    1: lambda a, b: "Wrong LZW header. Magic bytes don't match. 0x%02x 0x%02x" % (a, b),
    2: lambda a, b: "Stream compressed with %d bits, but decompression can only handle 16 bits." % a,
    3: lambda a, b: "Unsupported bits set in the header.",
    4: lambda a, b: "corrupt input: %d > 255" % a,
    5: lambda a, b: "corrupt input: code=%d, freeEnt=%d" % (a, b),
}


def lib():
    global _L
    if _L is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = _SO + ".%d" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", tmp, _SRC])
            os.replace(tmp, _SO)
        L = C.CDLL(_SO)
        L.lzw_model_decode.restype = C.c_int
        L.lzw_model_decode.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                       C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        L.lzw_model_encode.restype = C.c_int64
        L.lzw_model_encode.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_int64]
        _L = L
    return _L


class Result:
    """kind 0: decoded to the end; otherwise the exception (kind, a, b).  out: the bytes the successful Reads returned;
    decoded: the bytes in front of the code that threw (what a Read of one byte at a time gets before the exception)."""

    def __init__(self, kind, a, b, out, decoded):
        self.kind, self.a, self.b, self.out, self.decoded = kind, a, b, out, decoded

    @property
    def message(self):
        return MESSAGES[self.kind](self.a, self.b) if self.kind in MESSAGES else None

    def __repr__(self):
        return "Result(kind=%d, a=%d, b=%d, %d bytes, decoded=%d)" % (self.kind, self.a, self.b, len(self.out), self.decoded)


def decode(data, read_sizes=None, out_chunk=0, cap=None):
    """LzwInputStream over `data`: the base stream's k-th Read after the header returns at most read_sizes[k % len] bytes;
    the caller reads out_chunk bytes per Read (0: 1 MiB)."""
    L = lib()
    a = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(1, np.uint8)
    sz = np.ascontiguousarray(read_sizes if read_sizes else [0], dtype=np.int32)
    cap = cap if cap is not None else max(1 << 16, 64 * len(data))
    while True:
        out = np.empty(cap + 1, np.uint8)
        dl, dc, ea, eb = C.c_int64(), C.c_int64(), C.c_int32(), C.c_int32()
        k = L.lzw_model_decode(a.ctypes.data, len(data), sz.ctypes.data, len(read_sizes) if read_sizes else 0, out_chunk,
                               out.ctypes.data, cap, C.byref(dl), C.byref(dc), C.byref(ea), C.byref(eb))
        if dl.value <= cap:
            return Result(k, ea.value, eb.value, out[:dl.value].tobytes(), dc.value)
        cap = dl.value


def encode(data, max_bits=16, block=True, clear_every=0, ratio_clear=True):
    """a compress(1)-format stream of `data`"""
    L = lib()
    a = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(1, np.uint8)
    cap = 3 + 2 * len(data) + 64
    while True:
        out = np.empty(cap, np.uint8)
        n = L.lzw_model_encode(a.ctypes.data, len(data), max_bits, 1 if block else 0, clear_every, 1 if ratio_clear else 0,
                               out.ctypes.data, cap)
        if n <= cap:
            return out[:n].tobytes()
        cap = n


class BitWriter:
    """hand-built .Z streams: codes LSB-first at a chosen width, with the decoder's padding to whole groups"""

    def __init__(self, max_bits=16, block=True, flags=None):
        self.out = bytearray([0x1F, 0x9D, flags if flags is not None else (max_bits | (0x80 if block else 0))])
        self.bit = 0
        self.group = 0

    def code(self, c, n):
        for k in range(n):
            byte = 3 + ((self.bit + k) >> 3)
            while len(self.out) <= byte:
                self.out.append(0)
            if (c >> k) & 1:
                self.out[byte] |= 1 << ((self.bit + k) & 7)
        self.bit += n
        return self

    def pad(self, n):
        """round the position up to a whole group of n-bit codes, counted from where the current width began"""
        g = 8 * n
        self.bit = self.group + (self.bit - self.group + g - 1) // g * g
        self.group = self.bit
        return self

    def bytes(self):
        return bytes(self.out[:3 + (self.bit + 7) // 8])
