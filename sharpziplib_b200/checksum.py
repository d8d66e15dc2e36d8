"""Crc32 / Adler32 / BZip2Crc -- mirrors of Checksum/Crc32.cs:47-171, Checksum/Adler32.cs:56-161 and
Checksum/BZip2Crc.cs:43-170 (IChecksum: Reset, Value, Update).  The reduction runs on the GPU (b200z_checksum.cu); the
object only keeps the running Value."""
import ctypes as C

import numpy as np

from . import _lib


def _as_u8(data, offset=0, count=None):
    a = data if isinstance(data, np.ndarray) else np.frombuffer(data, dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    if count is None:
        count = a.size - offset
    if offset < 0 or count < 0 or offset + count > a.size:
        raise ValueError("offset/count")
    return a[offset:offset + count]


class _Checksum:
    _INIT = 0
    _fn = None

    def __init__(self):
        self._value = self._INIT

    def Reset(self):
        self._value = self._INIT

    @property
    def Value(self):
        return self._value

    def Update(self, data, offset=0, count=None):
        """Update(int) takes the low 8 bits (Crc32.cs:100, Adler32.cs:96, BZip2Crc.cs:99); Update(bytes/ArraySegment) the
        whole span."""
        if isinstance(data, int):
            data = bytes([data & 0xFF])
        a = _as_u8(data, offset, count)
        v = C.c_uint32(self._value)
        fn = getattr(_lib.lib(), self._fn)
        _lib.raise_for(fn(a.ctypes.data if a.size else None, a.size, C.byref(v)))
        self._value = v.value

    # pythonic aliases
    reset = Reset
    update = Update

    @property
    def value(self):
        return self._value


class Crc32(_Checksum):
    """CRC-32/ISO-HDLC: reflected 0xEDB88320, init/xorout 0xFFFFFFFF (Crc32.cs:50-59)."""
    _INIT = 0
    _fn = "b200z_crc32"


class BZip2Crc(_Checksum):
    """CRC-32/BZIP2: normal 0x04C11DB7, init/xorout 0xFFFFFFFF (BZip2Crc.cs:47-50).  Value is ~checkValue, so 0 after Reset."""
    _INIT = 0
    _fn = "b200z_bzip2crc"


class Adler32(_Checksum):
    """Adler-32, base 65521 (Adler32.cs:56)."""
    _INIT = 1
    _fn = "b200z_adler32"
