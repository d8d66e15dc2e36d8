"""LZW (.Z, Unix compress) decompression on the GPU: LzwInputStream (Lzw/LzwInputStream.cs), LZW batch plans and the batch
call.  Every byte is decoded by the kernels in csrc/b200z_lzw.cu."""
import ctypes as C

import numpy as np

from . import _lib
from .batch import _Plan, _ptr_array


class LzwException(_lib.SharpZipBaseException):
    """Mirror of ICSharpCode.SharpZipLib.Lzw.LzwException."""


# status detail -> the reference's message, from the numbers the run reports (INTEGRATION.md §2)
_MESSAGES = {
    32: lambda v: "Wrong LZW header. Magic bytes don't match. 0x%02x 0x%02x" % (v >> 8, v & 0xFF),
    33: lambda v: "Stream compressed with %d bits, but decompression can only handle 16 bits." % v,
    34: lambda v: "Unsupported bits set in the header.",
    35: lambda v: "corrupt input: %d > 255" % v,
    36: lambda v: "corrupt input: code=%d, freeEnt=%d" % (v >> 16, v & 0xFFFF),
}


def error_for(status, value):
    """the exception the reference throws for a stream's status and reported numbers (None for a good stream)"""
    code, detail = status & 0xFF, (status >> 8) & 0xFF
    if code == _lib.OK:
        return None
    if code == _lib.E_DATA:
        return LzwException(_MESSAGES[detail](int(value)))
    if code == _lib.E_INTERNAL:  # the reference fails with an index or Array.Copy exception, not an LzwException
        return RuntimeError("LZW stream: the reference fails with a non-SharpZip exception (status detail %d)" % detail)
    if code == _lib.E_NOMEM:
        return MemoryError("LZW stream: the output does not fit its capacity")
    return RuntimeError("b200z status %d" % status)


class LzwPlan(_Plan):
    """n independent .Z streams of comp_lens bytes (header included) decoding into at most out_caps bytes each.  run()
    takes d_check as the per-stream numbers of the error messages; stats() gives epochs, codes and the longest string."""

    def __init__(self, comp_lens, out_caps):
        cl = np.ascontiguousarray(comp_lens, dtype=np.int64)
        oc = np.ascontiguousarray(out_caps, dtype=np.int64)
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_lzw_plan_create(cl.size, cl.ctypes.data, oc.ctypes.data, C.byref(h)))
        self.comp_lens, self.out_caps = cl, oc
        super().__init__(h, cl.size)

    def stats(self, stream=None):
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        v = np.zeros(3, dtype=np.uint32)
        _lib.raise_for(_lib.lib().b200z_plan_get_stats(self._h, v.ctypes.data, 3, s.cuda_stream))
        return dict(zip(("epochs", "codes", "longest"), (int(x) for x in v)))


def _run(ins, lens, caps, devices):
    n = len(ins)
    outs = [np.empty(int(c) + 1, dtype=np.uint8) for c in caps]
    out_len = np.zeros(n, dtype=np.int64)
    in_used = np.zeros(n, dtype=np.int64)
    value = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    if devices is not None:
        dv = np.ascontiguousarray(devices, dtype=np.int32)
        rc = _lib.lib().b200z_lzw_batch_multi(dv.ctypes.data, dv.size, _ptr_array(ins), lens.ctypes.data, n, _ptr_array(outs),
                                              caps.ctypes.data, out_len.ctypes.data, in_used.ctypes.data, value.ctypes.data,
                                              status.ctypes.data)
    else:
        rc = _lib.lib().b200z_lzw_batch(_ptr_array(ins), lens.ctypes.data, n, _ptr_array(outs), caps.ctypes.data,
                                        out_len.ctypes.data, in_used.ctypes.data, value.ctypes.data, status.ctypes.data)
    if rc in (_lib.E_CUDA, _lib.E_ARG, _lib.E_STATE, _lib.E_UNSUPPORTED):
        _lib.raise_for(rc)
    return outs, out_len, in_used, value, status


def lzw_batch(buffers, out_caps=None, devices=None):
    """Decode .Z streams (b200z_lzw_batch; devices: b200z_lzw_batch_multi over those GPUs).  .Z has no size field: a stream
    whose output does not fit its capacity (default 4 x its length + 64 KiB) reports the size it needs, and those streams are
    run once more with it.  Returns (outputs, status, value): outputs[i] is the bytes in front of stream i's first bad code,
    status[i] = code | detail << 8, value[i] the numbers of its error message (error_for turns both into the exception)."""
    ins = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8)) for b in buffers]
    lens = np.array([a.size for a in ins], dtype=np.int64)
    caps = (np.ascontiguousarray(out_caps, dtype=np.int64).copy() if out_caps is not None
            else np.array([4 * l + 65536 for l in lens], dtype=np.int64))
    outs, out_len, _, value, status = _run(ins, lens, caps, devices)
    res = [outs[i][:out_len[i]].tobytes() for i in range(len(ins))]
    again = [i for i in range(len(ins)) if (status[i] & 0xFF) == _lib.E_NOMEM]
    if again:
        sub = [ins[i] for i in again]
        o2, l2, _, v2, s2 = _run(sub, lens[again], out_len[again].copy(), devices)
        for k, i in enumerate(again):
            res[i], status[i], value[i] = o2[k][:l2[k]].tobytes(), s2[k], v2[k]
    return res, status, value


class LzwInputStream:
    """Mirror of LzwInputStream (Lzw/LzwInputStream.cs).  The header is one Read of 3 bytes from the base stream, as
    ParseHeader (:342) does.  At the first Read the handle reads the rest of the base stream to its end, decodes it in one
    device run and holds the whole output on the host; it then hands out bytes and raises where the reference would: on the
    first Read that reaches the failing code, after every byte in front of it was handed out.  Streams are not resumed with
    bounded memory."""

    def __init__(self, baseInputStream):
        self.baseInputStream = baseInputStream
        self.IsStreamOwner = True
        self._out = None
        self._err = None
        self._pos = 0
        self._closed = False

    def _decode(self):
        hdr = self.baseInputStream.read(3) or b""  # one Read: a short read leaves zeros in the header
        hdr = bytes(hdr) + bytes(3 - len(hdr))
        rest = bytearray()
        while True:
            b = self.baseInputStream.read(1 << 20)
            if not b:
                break
            rest += b
        outs, status, value = lzw_batch([hdr + bytes(rest)])
        self._out, self._err = outs[0], error_for(int(status[0]), int(value[0]))
        st = int(status[0])
        self._header_error = (st & 0xFF, st >> 8 & 0xFF) in ((_lib.E_DATA, 32), (_lib.E_DATA, 33), (_lib.E_DATA, 34), (_lib.E_INTERNAL, 1))

    def Read(self, buffer, offset, count):
        if self._out is None:
            self._decode()
        if count <= 0:
            if self._err is not None and self._header_error:  # ParseHeader runs before the count is looked at
                raise self._err
            return 0
        left = len(self._out) - self._pos
        if self._err is not None and count > left:
            raise self._err
        k = min(count, left)
        buffer[offset:offset + k] = self._out[self._pos:self._pos + k]
        self._pos += k
        return k

    def ReadByte(self):
        b = bytearray(1)
        return b[0] if self.Read(b, 0, 1) == 1 else -1

    def read(self, size=-1):
        """file-like read: `size` bytes by one Read (all the rest when size < 0)"""
        if self._out is None:
            self._decode()
        n = len(self._out) - self._pos + (1 if self._err is not None else 0) if size is None or size < 0 else size
        b = bytearray(n)
        k = self.Read(b, 0, n)
        return bytes(b[:k])

    def Close(self):
        if not self._closed:
            self._closed = True
            if self.IsStreamOwner and hasattr(self.baseInputStream, "close"):
                self.baseInputStream.close()

    close = Close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Close()
