"""Deflater / Inflater -- host mirrors of Zip/Compression/Deflater.cs and Zip/Compression/Inflater.cs over the
streaming handles of libb200z.so.  Member names follow the reference; snake_case aliases are provided."""
import ctypes as C

import numpy as np

from . import _lib
from .checksum import _as_u8

INT32_MAX = 0x7FFFFFFF  # SetInput's count is a C# int, and an int32_t in the C-ABI


def _input(data, offset, count):
    """the span SetInput hands to the library; a longer one is refused rather than cut to its count's low 32 bits"""
    a = _as_u8(data, offset, count)
    if a.size > INT32_MAX:
        raise ValueError("count: %d bytes in one SetInput (at most %d)" % (a.size, INT32_MAX))
    return a


class DeflateStrategy:
    """Zip/Compression/DeflaterEngine.cs:9-28"""
    Default = 0
    Filtered = 1
    HuffmanOnly = 2


class Deflater:
    """new Deflater(level, noZlibHeaderOrFooter) -- Deflater.cs:149-195.  level -1 means 6; 0..9 otherwise."""

    BEST_COMPRESSION = 9
    BEST_SPEED = 1
    DEFAULT_COMPRESSION = -1
    NO_COMPRESSION = 0
    DEFLATED = 8

    def __init__(self, level=-1, noZlibHeaderOrFooter=False):
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_deflater_create(level, 1 if noZlibHeaderOrFooter else 0, C.byref(h)))
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            _lib.lib().b200z_deflater_destroy(h)
            self._h = None

    def Reset(self):  # :204
        _lib.raise_for(_lib.lib().b200z_deflater_reset(self._h))

    def SetLevel(self, level):  # :349
        _lib.raise_for(_lib.lib().b200z_deflater_set_level(self._h, level))

    def GetLevel(self):  # :371
        v = C.c_int(0)
        _lib.raise_for(_lib.lib().b200z_deflater_get_level(self._h, C.byref(v)))
        return v.value

    def SetStrategy(self, strategy):  # :385
        _lib.raise_for(_lib.lib().b200z_deflater_set_strategy(self._h, strategy))

    def SetDictionary(self, dictionary, index=0, count=None):  # :534/:559
        a = _as_u8(dictionary, index, count)
        _lib.raise_for(_lib.lib().b200z_deflater_set_dictionary(self._h, a.ctypes.data, a.size))

    def SetInput(self, input, offset=0, count=None):  # :308/:331
        a = _input(input, offset, count)
        _lib.raise_for(_lib.lib().b200z_deflater_set_input(self._h, a.ctypes.data if a.size else None, a.size))

    def Flush(self):  # :252
        _lib.raise_for(_lib.lib().b200z_deflater_flush(self._h))

    def Finish(self):  # :262
        _lib.raise_for(_lib.lib().b200z_deflater_finish(self._h))

    def Deflate(self, output, offset=0, length=None):
        """Deflate(byte[] output, int offset, int length) -> bytes written (:427).  `output` is a writable buffer
        (bytearray / numpy uint8)."""
        buf = np.frombuffer(output, dtype=np.uint8) if not isinstance(output, np.ndarray) else output
        if not buf.flags.writeable:
            raise TypeError("Deflate() writes into `output`: pass a bytearray / writable array, not bytes")
        if length is None:
            length = buf.size - offset
        if offset < 0 or length < 0 or offset + length > buf.size:
            raise ValueError("offset/length")
        p = C.c_int32(0)
        _lib.raise_for(_lib.lib().b200z_deflater_deflate(self._h, buf.ctypes.data + offset, length, C.byref(p)))
        return p.value

    @property
    def IsFinished(self):  # :271
        v = C.c_int(0)
        _lib.raise_for(_lib.lib().b200z_deflater_is_finished(self._h, C.byref(v)))
        return bool(v.value)

    @property
    def IsNeedingInput(self):  # :285
        v = C.c_int(0)
        _lib.raise_for(_lib.lib().b200z_deflater_needs_input(self._h, C.byref(v)))
        return bool(v.value)

    @property
    def TotalIn(self):  # :226
        v = C.c_int64(0)
        _lib.raise_for(_lib.lib().b200z_deflater_total_in(self._h, C.byref(v)))
        return v.value

    @property
    def TotalOut(self):  # :237
        v = C.c_int64(0)
        _lib.raise_for(_lib.lib().b200z_deflater_total_out(self._h, C.byref(v)))
        return v.value

    @property
    def Adler(self):  # :215
        v = C.c_uint32(0)
        _lib.raise_for(_lib.lib().b200z_deflater_adler(self._h, C.byref(v)))
        return v.value


class Inflater:
    """new Inflater(noHeader) -- Inflater.cs:156-180."""

    def __init__(self, noHeader=False):
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_inflater_create(1 if noHeader else 0, C.byref(h)))
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            _lib.lib().b200z_inflater_destroy(h)
            self._h = None

    def Reset(self):  # :188
        _lib.raise_for(_lib.lib().b200z_inflater_reset(self._h))

    def SetDictionary(self, buffer, index=0, count=None):  # :563/:589
        a = _as_u8(buffer, index, count)
        _lib.raise_for(_lib.lib().b200z_inflater_set_dictionary(self._h, a.ctypes.data, a.size))

    def SetInput(self, buffer, index=0, count=None):  # :629/:653
        a = _input(buffer, index, count)
        _lib.raise_for(_lib.lib().b200z_inflater_set_input(self._h, a.ctypes.data if a.size else None, a.size))

    def Inflate(self, buffer, offset=0, count=None):
        """Inflate(byte[] buffer, int offset, int count) -> bytes produced (:715); argument checks as :717-735."""
        if buffer is None:
            raise ValueError("buffer")
        buf = np.frombuffer(buffer, dtype=np.uint8) if not isinstance(buffer, np.ndarray) else buffer
        if not buf.flags.writeable:
            raise TypeError("Inflate() writes into `buffer`: pass a bytearray / writable array, not bytes")
        if count is None:
            count = buf.size - offset
        if count < 0:
            raise ValueError("count cannot be negative")
        if offset < 0:
            raise ValueError("offset cannot be negative")
        if offset + count > buf.size:
            raise ValueError("count exceeds buffer bounds")
        p = C.c_int32(0)
        _lib.raise_for(_lib.lib().b200z_inflater_inflate(self._h, buf.ctypes.data + offset, count, C.byref(p)))
        return p.value

    def _flag(self, name):
        v = C.c_int(0)
        _lib.raise_for(getattr(_lib.lib(), name)(self._h, C.byref(v)))
        return bool(v.value)

    @property
    def IsNeedingInput(self):  # :783
        return self._flag("b200z_inflater_needs_input")

    @property
    def IsNeedingDictionary(self):  # :794
        return self._flag("b200z_inflater_needs_dictionary")

    @property
    def IsFinished(self):  # :806
        return self._flag("b200z_inflater_is_finished")

    @property
    def RemainingInput(self):  # :878
        v = C.c_int32(0)
        _lib.raise_for(_lib.lib().b200z_inflater_remaining_input(self._h, C.byref(v)))
        return v.value

    @property
    def TotalIn(self):  # :862
        v = C.c_int64(0)
        _lib.raise_for(_lib.lib().b200z_inflater_total_in(self._h, C.byref(v)))
        return v.value

    @property
    def TotalOut(self):  # :848
        v = C.c_int64(0)
        _lib.raise_for(_lib.lib().b200z_inflater_total_out(self._h, C.byref(v)))
        return v.value

    @property
    def Adler(self):  # :823
        v = C.c_uint32(0)
        _lib.raise_for(_lib.lib().b200z_inflater_adler(self._h, C.byref(v)))
        return v.value

    def stats(self):
        """diagnostics since construction / Reset (b200z_inflater_get_stats; not in the reference): device runs, output bytes
        the runs produced (re-decoded bytes counted again), most compressed and most output bytes held at once"""
        v = np.zeros(4, dtype=np.int64)
        _lib.raise_for(_lib.lib().b200z_inflater_get_stats(self._h, v.ctypes.data, 4))
        return dict(zip(("runs", "decoded", "max_comp_held", "max_out_held"), (int(x) for x in v)))
