"""Stream adapters -- host mirrors of Streams/DeflaterOutputStream.cs, Streams/InflaterInputStream.cs and the GZip
framing of GZip/GzipOutputStream.cs / GzipInputStream.cs.  These stay on the host in the reference's design too
(SURVEY.md 8b); they drive the Deflater / Inflater handles exactly as the C# code does."""
import io
import struct

from ._lib import SharpZipBaseException
from .checksum import Crc32, _as_u8
from .codec import INT32_MAX, Deflater, Inflater


class DeflaterOutputStream:
    """DeflaterOutputStream(Stream baseOutputStream, Deflater deflater, int bufferSize = 512) -- :49-93."""

    def __init__(self, baseOutputStream, deflater=None, bufferSize=512):
        if baseOutputStream is None:
            raise ValueError("baseOutputStream")
        if bufferSize < 512:
            raise ValueError("bufferSize")  # :79-82
        self.baseOutputStream_ = baseOutputStream
        self.deflater_ = deflater if deflater is not None else Deflater()
        self.buffer_ = bytearray(bufferSize)
        self.IsStreamOwner = True
        self._closed = False

    def Finish(self):  # :100-139
        self.deflater_.Finish()
        while not self.deflater_.IsFinished:
            n = self.deflater_.Deflate(self.buffer_, 0, len(self.buffer_))
            if n <= 0:
                break
            self.baseOutputStream_.write(bytes(self.buffer_[:n]))
        if not self.deflater_.IsFinished:
            raise SharpZipBaseException("Can't deflate all input?")
        if hasattr(self.baseOutputStream_, "flush"):
            self.baseOutputStream_.flush()

    def _deflate(self, flushing):  # DeflateSyncOrAsync :245-275
        while flushing or not self.deflater_.IsNeedingInput:
            n = self.deflater_.Deflate(self.buffer_, 0, len(self.buffer_))
            if n <= 0:
                break
            self.baseOutputStream_.write(bytes(self.buffer_[:n]))
        if not self.deflater_.IsNeedingInput:
            raise SharpZipBaseException("DeflaterOutputStream can't deflate all input?")

    def Write(self, buffer, offset=0, count=None):  # :506-510
        a = _as_u8(buffer, offset, count)
        # a C# caller cannot pass more than int.MaxValue bytes at once: a longer span goes as consecutive Writes of 1 GiB
        step = max(a.size, 1) if a.size <= INT32_MAX else 1 << 30
        for p in range(0, max(a.size, 1), step):
            self.deflater_.SetInput(a[p:p + step])
            self._deflate(False)

    def WriteByte(self, value):  # Stream.WriteByte -> Write of one byte (:495-504)
        self.Write(bytes([value & 0xFF]))

    def Flush(self):  # :388-393
        self.deflater_.Flush()
        self._deflate(True)
        if hasattr(self.baseOutputStream_, "flush"):
            self.baseOutputStream_.flush()

    def Close(self):  # Dispose :412-448
        if not self._closed:
            self._closed = True
            try:
                self.Finish()
            finally:
                if self.IsStreamOwner and hasattr(self.baseOutputStream_, "close"):
                    self.baseOutputStream_.close()

    write, flush, close = Write, Flush, Close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Close()


class InflaterInputStream:
    """InflaterInputStream(Stream baseInputStream, Inflater inflater, int bufferSize = 4096) -- :358-410."""

    def __init__(self, baseInputStream, inflater=None, bufferSize=4096):
        if baseInputStream is None:
            raise ValueError("baseInputStream")
        if bufferSize <= 0:
            raise ValueError("bufferSize")
        self.baseInputStream = baseInputStream
        self.inf = inflater if inflater is not None else Inflater()
        self._bufferSize = bufferSize
        self.IsStreamOwner = True

    def Fill(self):  # :486-498 + InflaterInputBuffer.Fill :115-144
        raw = self.baseInputStream.read(self._bufferSize)
        if not raw:
            raise SharpZipBaseException("Unexpected EOF")
        self.inf.SetInput(raw)

    def Read(self, buffer, offset=0, count=None):  # :658-690
        if count is None:
            count = len(buffer) - offset
        if self.inf.IsNeedingDictionary:
            raise SharpZipBaseException("Need a dictionary")
        remaining = count
        while True:
            n = self.inf.Inflate(buffer, offset, remaining)
            offset += n
            remaining -= n
            if remaining == 0 or self.inf.IsFinished:
                break
            if self.inf.IsNeedingInput:
                self.Fill()
            elif n == 0:
                raise SharpZipBaseException("Invalid input data")  # ZipException in the reference (:676)
        return count - remaining

    def read(self, n=-1):
        out = bytearray()
        chunk = bytearray(65536)
        while n < 0 or len(out) < n:
            want = len(chunk) if n < 0 else min(len(chunk), n - len(out))
            got = self.Read(chunk, 0, want)
            if got == 0:
                break
            out += chunk[:got]
        return bytes(out)

    def Close(self):
        if self.IsStreamOwner and hasattr(self.baseInputStream, "close"):
            self.baseInputStream.close()

    close = Close


class GZipOutputStream(DeflaterOutputStream):
    """GZipOutputStream(Stream baseOutputStream, int size = 4096) -- GZip/GzipOutputStream.cs:40-100.
    Header: 1F 8B 08 FLG MTIME(4, LE) XFL=0 OS=255 [FNAME 0] (:339-375, trap T15); footer CRC32 LE, ISIZE LE (:315-337)."""

    def __init__(self, baseOutputStream, size=4096, level=Deflater.DEFAULT_COMPRESSION):
        super().__init__(baseOutputStream, Deflater(level, True), size)
        self.crc = Crc32()
        self._state = "Header"
        self.ModifiedTime = None  # seconds since the Unix epoch, or None for "now"
        self._fileName = None
        self._total = 0

    @property
    def FileName(self):
        return self._fileName

    @FileName.setter
    def FileName(self, value):  # :121-139 (CleanFilename keeps what follows the last '/')
        self._fileName = value[value.rfind("/") + 1:] if value else None

    def SetLevel(self, level):  # :104-109
        if level < Deflater.BEST_SPEED:
            raise ValueError("level")
        self.deflater_.SetLevel(level)

    def GetLevel(self):
        return self.deflater_.GetLevel()

    def _header(self):
        import time
        mod = int(time.time()) if self.ModifiedTime is None else int(self.ModifiedTime)
        flags = 0x08 if self._fileName else 0
        h = bytes([0x1F, 0x8B, 0x08, flags]) + struct.pack("<I", mod & 0xFFFFFFFF) + bytes([0, 255])
        if self._fileName:
            try:
                nm = self._fileName.encode("cp1252")
            except UnicodeError:
                nm = self._fileName.encode("ascii", "replace")
            h += nm + b"\0"
        return h

    def _write_header(self):  # WriteHeader :380-386
        if self._state == "Header":
            self._state = "Footer"
            self.baseOutputStream_.write(self._header())

    def Write(self, buffer, offset=0, count=None):  # :156-178
        if self._state == "Header":
            self._write_header()
        if self._state != "Footer":
            raise RuntimeError("Write not permitted in current state")
        self.crc.Update(buffer, offset, count)
        n = (len(buffer) - offset) if count is None else count
        self._total += n
        super().Write(buffer, offset, count)

    def Flush(self):  # :245-268
        if self._state == "Header":
            self._write_header()
        super().Flush()

    def Finish(self):  # :276-291
        if self._state == "Header":
            self._write_header()
        if self._state == "Footer":
            self._state = "Finished"
            super().Finish()
            totalin = self.deflater_.TotalIn & 0xFFFFFFFF
            self.baseOutputStream_.write(struct.pack("<II", self.crc.Value & 0xFFFFFFFF, totalin))

    write, flush = Write, Flush


class GZipInputStream(InflaterInputStream):
    """Single/multi-member gzip reader -- GZip/GzipInputStream.cs:38-360.  Header parse (FEXTRA / FNAME / FCOMMENT / FHCRC),
    inflate, CRC-32 of the output and the CRC / ISIZE comparison with the footer all run on the device, one member per
    call of the batch ABI with B200Z_WRAP_GZIP (k_wrap_head, k_inflate, checksum kernel, k_wrap_tail); this class only
    loops over the members the way Read (:96-155) does: a header that fails after at least one complete member is
    trailing garbage and ends the stream quietly (:107-123), a member cut short hands out what was decoded and then
    raises."""

    MAX_MEMBER_OUTPUT = 1 << 32  # a member that inflates to more is refused (a 1 KiB gzip bomb asks for gigabytes otherwise)

    def __init__(self, baseInputStream, size=4096):
        super().__init__(baseInputStream, Inflater(True), size)
        self._data = None
        self._out = bytearray()
        self._served = 0
        self._error = None
        self._fileName = None

    def GetFilename(self):  # :160-163: the FNAME field of the (last read) member header
        self._decode()
        return self._fileName

    def _decode(self):
        if self._data is not None:
            return
        from . import _lib
        from .batch import inflate_batch
        d = self._data = memoryview(self.baseInputStream.read())  # (members are slices of one buffer, not copies)
        pos, completed = 0, False
        while pos < len(d):
            blob = d[pos:]
            cap = max(1 << 16, 8 * len(blob))
            while True:
                outs, used, st = inflate_batch([blob], [cap], raise_on_error=False, wrap=_lib.WRAP_GZIP)
                code, detail = int(st[0]) & 0xFF, int(st[0]) >> 8
                if code != _lib.E_NOMEM:
                    break
                if cap >= self.MAX_MEMBER_OUTPUT:
                    raise SharpZipBaseException("gzip member inflates to more than %d bytes (GZipInputStream.MAX_MEMBER_OUTPUT)" % self.MAX_MEMBER_OUTPUT)
                cap = min(cap * 8, self.MAX_MEMBER_OUTPUT)
            header_failed = int(used[0]) == 0 and (code == _lib.E_NEED_INPUT or (code == _lib.E_DATA and 14 <= detail <= 18))
            if code == _lib.OK:
                self._out += outs[0]
                if blob[3] & 0x08:  # FNAME: zero terminated, behind the optional FEXTRA (:248-270)
                    q = 10 + ((2 + (blob[10] | (blob[11] << 8))) if blob[3] & 0x04 else 0)
                    self._fileName = bytes(blob[q:q + bytes(blob[q:q + 65536]).index(0)]).decode("cp1252", "replace")
                else:
                    self._fileName = None
                pos += int(used[0])
                completed = True
                continue
            if header_failed and completed:
                break  # trailing garbage behind a complete member
            self._out += outs[0]  # whatever was decoded before the stream broke off
            msg = _lib.lib().b200z_last_error().decode("utf-8", "replace") if code == _lib.E_DATA else \
                ("EOS reading GZIP header" if header_failed else "Unexpected EOF")
            self._error = SharpZipBaseException(msg)
            break

    def Read(self, buffer, offset=0, count=None):  # :96-155
        self._decode()
        if count is None:
            count = len(buffer) - offset
        n = min(count, len(self._out) - self._served)
        if n == 0 and self._error is not None:
            err, self._error = self._error, None
            raise err
        buffer[offset:offset + n] = self._out[self._served:self._served + n]
        self._served += n
        return n

    def ReadByte(self):
        b = bytearray(1)
        return b[0] if self.Read(b, 0, 1) == 1 else -1

    def read(self, n=-1):
        self._decode()
        avail = len(self._out) - self._served
        if avail == 0 and self._error is not None:
            err, self._error = self._error, None
            raise err
        k = avail if n < 0 else min(n, avail)
        r = bytes(self._out[self._served:self._served + k])
        self._served += k
        return r
