"""Batch plans over device tensors (what bench.py drives) and host-buffer batch helpers.

torch is used for device memory and streams only; every kernel launch happens inside libb200z.so.
"""
import ctypes as C

import numpy as np

from . import _lib


class _Plan:
    def __init__(self, handle, n):
        self._h = handle
        self.n = n
        L = _lib.lib()
        self.in_bytes = L.b200z_plan_in_bytes(handle)
        self.out_bytes = L.b200z_plan_out_bytes(handle)
        self.in_offsets = np.array([L.b200z_plan_in_offset(handle, i) for i in range(n)], dtype=np.int64)
        # where slot i's data starts (behind a history / preset dictionary, if the plan has one)
        self.data_offsets = np.array([L.b200z_plan_data_offset(handle, i) for i in range(n)], dtype=np.int64)
        self.out_offsets = np.array([L.b200z_plan_out_offset(handle, i) for i in range(n)], dtype=np.int64)
        self.workspace_bytes = L.b200z_plan_workspace_bytes(handle)
        self.launches = L.b200z_plan_launches(handle)

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().b200z_plan_destroy(h)
            except Exception:  # interpreter shutdown: the module globals may already be gone
                pass

    __del__ = close

    def set_timing(self, enable=True):
        _lib.raise_for(_lib.lib().b200z_plan_set_timing(self._h, 1 if enable else 0))

    def timings(self):
        """{kernel name: milliseconds} of the last run (call after synchronising the stream)."""
        names = C.create_string_buffer(1024)
        ms = (C.c_float * 32)()
        cnt = C.c_int32(0)
        _lib.raise_for(_lib.lib().b200z_plan_get_timings(self._h, names, 1024, ms, 32, C.byref(cnt)))
        keys = names.value.decode().split(";")[:cnt.value]
        return {k: float(ms[i]) for i, k in enumerate(keys)}

    def run(self, d_in, d_out, d_out_len, d_status, d_check=None, d_in_used=None, stream=None, stages=_lib.STAGE_ALL):
        """All arguments are CUDA torch tensors (uint8 blobs, int64 lengths, int32 status, uint32/int32 checks).
        Launches on `stream` (a torch.cuda.Stream) or the current stream; does not synchronise.
        stages: STAGE_SEARCH / STAGE_ENCODE run the two halves separately (b200z_plan_run_stages)."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        assert d_in.is_cuda and d_out.is_cuda and d_in.numel() >= self.in_bytes and d_out.numel() >= self.out_bytes
        rc = _lib.lib().b200z_plan_run_stages(self._h, d_in.data_ptr(), d_out.data_ptr(), d_out_len.data_ptr(),
                                              d_status.data_ptr(), d_check.data_ptr() if d_check is not None else None,
                                              d_in_used.data_ptr() if d_in_used is not None else None, stages, s.cuda_stream)
        _lib.raise_for(rc)


    def pack(self, d_out, d_out_len, d_packed, d_packed_off, stream=None):
        """streams of the last run back to back in d_packed; d_packed_off (int64, n + 1) gets starts and the total"""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        _lib.raise_for(_lib.lib().b200z_plan_pack(self._h, d_out.data_ptr(), d_out_len.data_ptr(), d_packed.data_ptr(),
                                                  d_packed_off.data_ptr(), s.cuda_stream))


class DeflatePlan(_Plan):
    """n independent streams, each what `new Deflater(level, true)` + SetInput(all) + Finish() would produce."""

    def __init__(self, in_lens, level=6, strategy=0, wrap=_lib.WRAP_RAW, end_mode=_lib.END_FINISH, dict_lens=None,
                 chunk_lens=None, history=None, entry=None, state=None, undrained=None):
        """dict_lens: per-stream preset-dictionary bytes (Deflater.SetDictionary; at most 32506, the reference keeps the
        dictionary's tail) stored in the input slot directly in front of the stream's data.
        chunk_lens: per stream, the sizes of the SetInput calls that deliver its data (each followed by Deflate() until
        IsNeedingInput, as DeflaterOutputStream.Write does); levels 0-4 depend on it (SURVEY.md trap T9), 5-9 ignore it.
        history: (hist_lens, pos_bases, bit_bases[, masks]) -- levels 5-9, the stream goes on behind earlier runs
        (B200Z_HIST_CONTINUE); pos_bases are the data's stream offsets, of any size, bit_bases the bits (0..7) the previous
        run left in its last byte, masks per stream the history positions that are not in the hash chains (default: none,
        which is what a cut leaves).
        end_mode=END_NONE: an open run, see cut().
        entry: per stream (prev_available, match_len, match_dist), the parse state to start from (set_entry).
        state (levels 0-4): the engine state carried between the runs of a stream -- at levels 1-4 n CUDA uint8 tensors of
        engine_state_bytes() each (head[], prev[], DeflateFast's scalars, written by the run), at level 0 a uint8 array of
        16 * n bytes (b200z_stored_state[n], overwritten when the plan is made).  With history the stream goes on from it;
        history and chunk_lens may then come together.  undrained: per stream, Flush() / Finish() follows the last SetInput
        without a Deflate() call in between."""
        lens = np.ascontiguousarray(in_lens, dtype=np.int64)
        n = lens.size
        kind, hl, pb, bb, masks = _lib.HIST_NONE, None, None, None, None
        if history is not None:
            kind, hl, pb = _lib.HIST_CONTINUE, np.ascontiguousarray(history[0], np.int64), np.ascontiguousarray(history[1], np.int64)
            bb = np.ascontiguousarray(history[2], dtype=np.int32)
            assert hl.size == n and pb.size == n and bb.size == n
            marr = None  # (with a state and no masks the library flags the last two history positions)
            if len(history) > 3:
                marr = [np.frombuffer(bytes(m) + b"\0", np.uint8) for m in history[3]]
            elif state is None:  # nothing flagged: what a cut leaves
                marr = [np.zeros(max(int(x), 1), np.uint8) for x in hl]
            masks = None if marr is None else _ptr_array(marr)
        elif dict_lens is not None:
            kind, hl = _lib.HIST_DICTIONARY, np.ascontiguousarray(dict_lens, dtype=np.int64)
        if chunk_lens is None and state is not None:
            chunk_lens = [[int(x)] for x in lens]  # one SetInput with everything
        counts = chunks = und = eng = st = None
        if chunk_lens is not None:
            assert len(chunk_lens) == n
            arrs = [np.ascontiguousarray(c, dtype=np.int64) for c in chunk_lens]
            counts, chunks = np.array([a.size for a in arrs], dtype=np.int32), _ptr_array(arrs)
        if undrained is not None:
            und = np.ascontiguousarray(undrained, dtype=np.int32)
        if state is not None and level == 0:
            assert isinstance(state, np.ndarray) and state.dtype == np.uint8 and state.size == 16 * n
            st = state.ctypes.data
        elif state is not None:
            assert len(state) == n
            eng = (C.c_void_p * n)(*[t.data_ptr() for t in state])
        self._state = state  # (levels 0-4: the plan and its runs write it)
        addr = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        ref = lambda a: None if a is None else C.addressof(a)  # noqa: E731
        hs = _lib.History(kind, 0, addr(hl), addr(pb), addr(bb), ref(masks), addr(counts), ref(chunks), addr(und), ref(eng), st)
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_deflate_plan_create_ex(n, lens.ctypes.data, level, strategy, wrap, end_mode,
                                                              C.addressof(hs), C.byref(h)))
        self.dict_lens = np.zeros(n, dtype=np.int64) if hl is None else hl
        self.in_lens = lens
        self.level = level
        super().__init__(h, n)
        if entry is not None:
            self.set_entry(entry)

    def set_entry(self, entry):
        """per stream (prev_available, match_len, match_dist): the parse state the next runs start from"""
        assert len(entry) == self.n
        arr = (_lib.ParseEntry * max(self.n, 1))(*[_lib.ParseEntry(*map(int, e)) for e in entry])
        _lib.raise_for(_lib.lib().b200z_deflate_plan_set_entry(self._h, arr))

    def cut(self, stream=None):
        """After an END_NONE run: (covered, entries) -- per stream the data bytes in front of the first block not written
        (the next run's data starts there) and the (prev_available, match_len, match_dist) to enter that run with.  At
        levels 0-4 (covered, calls): the state is in the plan's `state`, and calls[i] is the SetInput call of chunk_lens[i]
        the cut fell into -- the next run's calls are the rest of it from `covered` on, then the ones behind it.
        Synchronises the stream."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        covered = np.zeros(self.n, dtype=np.int64)
        if self.level <= 4:
            calls = np.zeros(max(self.n, 1), dtype=np.int32)
            _lib.raise_for(_lib.lib().b200z_deflate_plan_get_cut(self._h, covered.ctypes.data, None, s.cuda_stream))
            _lib.raise_for(_lib.lib().b200z_deflate_plan_get_cut_call(self._h, calls.ctypes.data, s.cuda_stream))
            return covered, [int(c) for c in calls[:self.n]]
        arr = (_lib.ParseEntry * max(self.n, 1))()
        _lib.raise_for(_lib.lib().b200z_deflate_plan_get_cut(self._h, covered.ctypes.data, arr, s.cuda_stream))
        return covered, [(e.prev_available, e.match_len, e.match_dist) for e in arr[:self.n]]


class InflatePlan(_Plan):
    """n independent raw deflate streams of comp_lens bytes decoding into at most out_caps bytes each."""

    def __init__(self, comp_lens, out_caps, wrap=_lib.WRAP_RAW, dict_lens=None):
        cl = np.ascontiguousarray(comp_lens, dtype=np.int64)
        oc = np.ascontiguousarray(out_caps, dtype=np.int64)
        h = C.c_void_p()
        dl = None if dict_lens is None else np.ascontiguousarray(dict_lens, dtype=np.int64)
        _lib.raise_for(_lib.lib().b200z_inflate_plan_create_ex(cl.size, cl.ctypes.data, oc.ctypes.data, wrap,
                                                              None if dl is None else dl.ctypes.data, C.byref(h)))
        self.dict_lens = dl
        self.comp_lens, self.out_caps = cl, oc
        super().__init__(h, cl.size)

    def set_start_bits(self, start_bits):
        """Raw plans: stream i's first block header starts at bit start_bits[i] (0..7) of its first compressed byte --
        decoding a stream on from a restart point, with the window image passed as the dictionary."""
        sb = np.ascontiguousarray(start_bits, dtype=np.int32)
        assert sb.size == self.n
        _lib.raise_for(_lib.lib().b200z_inflate_plan_set_start_bits(self._h, sb.ctypes.data))

    def set_resume(self, start_bits, skip_bits):
        """Raw plans: stream i enters a Huffman block in its middle.  Its slot holds the block's header from bit start_bits[i]
        (0..7) of its first compressed byte, then the compressed bytes from the resume point on; decoding goes on at bit
        skip_bits[i] of the slot (0: no jump, a plain start bit).  The window image is passed as the dictionary."""
        sb = np.ascontiguousarray(start_bits, dtype=np.int32)
        kb = np.ascontiguousarray(skip_bits, dtype=np.int64)
        assert sb.size == self.n and kb.size == self.n
        _lib.raise_for(_lib.lib().b200z_inflate_plan_set_resume(self._h, sb.ctypes.data, kb.ctypes.data))

    def stats(self, stream=None):
        """diagnostics of the last run (b200z_plan_get_stats): finder survivors, segments, round slots, blocks, rounds, passes,
        streams handed back to the serial kernel, pipeline in use"""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        v = np.zeros(8, dtype=np.uint32)
        _lib.raise_for(_lib.lib().b200z_plan_get_stats(self._h, v.ctypes.data, 8, s.cuda_stream))
        names = ("finder_survivors", "segments", "round_slots", "blocks", "rounds", "passes", "handed_back", "parallel")
        return dict(zip(names, (int(x) for x in v)))

    def restart_points(self, stream=None):
        """(bit, out_pos) int64 arrays of the last run: where the last block header each stream's decoder reached lies
        (bits from the first compressed byte of the slot; output bytes in front of it).  Synchronises the stream."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        bit = np.zeros(self.n, dtype=np.int64)
        pos = np.zeros(self.n, dtype=np.int64)
        _lib.raise_for(_lib.lib().b200z_plan_get_restart_points(self._h, bit.ctypes.data, pos.ctypes.data, s.cuda_stream))
        return bit, pos

    def resume_points(self, stream=None):
        """(hdr_bit, body_bit, sym_bit, out_pos) int64 arrays of the last run (bits from the first compressed byte of the
        slot): the header of the block each stream stopped in, where that header ends, the first symbol not decoded and the
        output bytes in front of it.  Inside the block only for a stream that stopped in a Huffman block; otherwise the three
        bits are the restart point.  Synchronises the stream."""
        import torch
        s = stream if stream is not None else torch.cuda.current_stream()
        v = [np.zeros(self.n, dtype=np.int64) for _ in range(4)]
        _lib.raise_for(_lib.lib().b200z_plan_get_resume_points(self._h, *(a.ctypes.data for a in v), s.cuda_stream))
        return tuple(v)


class Pipeline:
    """Host-buffer pipeline (b200z_*_pipeline_*): submit() stages one batch from host memory and enqueues upload and kernels
    without waiting, collect() waits for the oldest batch and hands the produced bytes to host memory.  `ins` / `outs` are
    sequences of integer host addresses (ctypes / numpy / torch data pointers), one per stream."""

    def __init__(self, handle, n, depth):
        self._h, self.n, self.depth = handle, n, depth
        self.out_len = np.zeros(n, dtype=np.int64)
        self.in_used = np.zeros(n, dtype=np.int64)
        self.check = np.zeros(n, dtype=np.uint32)
        self.status = np.zeros(n, dtype=np.int32)

    @classmethod
    def deflate(cls, in_lens, level=6, strategy=0, wrap=_lib.WRAP_RAW, end_mode=_lib.END_FINISH, depth=2):
        lens = np.ascontiguousarray(in_lens, dtype=np.int64)
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_deflate_pipeline_create(lens.size, lens.ctypes.data, level, strategy, wrap, end_mode, depth, C.byref(h)))
        return cls(h, lens.size, depth)

    @classmethod
    def inflate(cls, comp_lens, out_caps, wrap=_lib.WRAP_RAW, depth=2):
        cl = np.ascontiguousarray(comp_lens, dtype=np.int64)
        oc = np.ascontiguousarray(out_caps, dtype=np.int64)
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_inflate_pipeline_create(cl.size, cl.ctypes.data, oc.ctypes.data, wrap, depth, C.byref(h)))
        return cls(h, cl.size, depth)

    @staticmethod
    def pointers(addresses):
        return (C.c_void_p * len(addresses))(*[int(a) if a else None for a in addresses])

    def submit(self, in_ptrs):
        _lib.raise_for(_lib.lib().b200z_pipeline_submit(self._h, in_ptrs))

    def collect(self, out_ptrs, out_caps, raise_on_error=True):
        rc = _lib.lib().b200z_pipeline_collect(self._h, out_ptrs, out_caps.ctypes.data, self.out_len.ctypes.data, self.in_used.ctypes.data,
                                              self.check.ctypes.data, self.status.ctypes.data)
        if raise_on_error or rc in (_lib.E_CUDA, _lib.E_ARG, _lib.E_STATE):
            _lib.raise_for(rc)
        return rc

    @property
    def in_flight(self):
        return int(_lib.lib().b200z_pipeline_in_flight(self._h))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().b200z_pipeline_destroy(h)
            except Exception:
                pass

    __del__ = close


def _ptr_array(arrs):
    return (C.c_void_p * len(arrs))(*[a.ctypes.data if a.size else None for a in arrs])


class DeflaterSet:
    """n independent Deflater streams of one level / strategy / wrap that arrive in pieces, run together on the device
    (b200z_deflate_streams_*): what n Deflater objects behind DeflaterOutputStream (GZipOutputStream for WRAP_GZIP) do,
    with one device pass per write() instead of one per stream."""
    NOTHING, FLUSH, FINISH = 0, 1, 2

    def __init__(self, n, level=6, strategy=0, wrap=_lib.WRAP_ZLIB):
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_deflate_streams_create(n, level, strategy, wrap, C.byref(h)))
        self._h = h
        self.n = n
        self.status = np.zeros(n, dtype=np.int32)  # per stream, of the last write()
        self._cap = np.full(n, 65536, dtype=np.int64)

    def write(self, buffers, ops=None):
        """Write(buffers[i]) on every stream, then ops[i]: 0 nothing, 1 Flush(), 2 Finish() (None: all 0).  An empty
        buffer with op 0 is no call, also for a finished stream.  A finished stream takes nothing else: its status is
        E_STATE, the others go on, and InvalidOperationException is raised after."""
        if len(buffers) != self.n or (ops is not None and len(ops) != self.n):
            raise ValueError("one buffer and one op per stream")
        ins = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8)) for b in buffers]
        lens = np.array([a.size for a in ins], dtype=np.int64)
        op = np.zeros(self.n, dtype=np.int32) if ops is None else np.ascontiguousarray(ops, dtype=np.int32)
        _lib.raise_for(_lib.lib().b200z_deflate_streams_write(self._h, _ptr_array(ins), lens.ctypes.data, op.ctypes.data,
                                                               self.status.ctypes.data))

    def read(self):
        """everything each stream has produced since the last read(), as a list of bytes"""
        parts = [[] for _ in range(self.n)]
        want = np.ones(self.n, dtype=bool)
        got = np.zeros(self.n, dtype=np.int64)
        while want.any():
            cap = np.where(want, self._cap, 0).astype(np.int64)
            outs = [np.empty(int(c), dtype=np.uint8) for c in cap]
            _lib.raise_for(_lib.lib().b200z_deflate_streams_read(self._h, _ptr_array(outs), cap.ctypes.data, got.ctypes.data))
            for i in np.nonzero(want)[0]:
                parts[i].append(outs[i][:got[i]].tobytes())
            want &= got == cap
            self._cap = np.where(want, np.minimum(self._cap * 4, 16 << 20), self._cap)
        return [b"".join(p) for p in parts]

    def checks(self):
        """per stream: Adler-32 (WRAP_ZLIB) or CRC-32 (WRAP_GZIP, WRAP_RAW_CRC32) of the bytes compressed so far"""
        v = np.zeros(self.n, dtype=np.uint32)
        _lib.raise_for(_lib.lib().b200z_deflate_streams_check(self._h, v.ctypes.data))
        return [int(x) for x in v]

    def stats(self):
        """{"runs": stream segments compressed, "plans": plans run, "held": most input bytes one stream held at once,
        "workspace": most device workspace one plan took}"""
        v = np.zeros(4, dtype=np.int64)
        _lib.raise_for(_lib.lib().b200z_deflate_streams_stats(self._h, v.ctypes.data, 4))
        return {"runs": int(v[0]), "plans": int(v[1]), "held": int(v[2]), "workspace": int(v[3])}

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().b200z_deflate_streams_destroy(h)
            except Exception:  # interpreter shutdown: the module globals may already be gone
                pass

    __del__ = close


class InflaterSet:
    """n independent Inflater streams of one wrap that arrive in pieces, decoded together on the device
    (b200z_inflate_streams_*): what n Inflater objects behind InflaterInputStream do, with one device pass per write()
    instead of one per stream.  wrap: WRAP_ZLIB, WRAP_RAW or WRAP_RAW_CRC32 (raw, with the CRC-32 a zip entry is checked
    against)."""

    def __init__(self, n, wrap=_lib.WRAP_ZLIB):
        h = C.c_void_p()
        _lib.raise_for(_lib.lib().b200z_inflate_streams_create(n, wrap, C.byref(h)))
        self._h = h
        self.n = n
        self.status = np.zeros(n, dtype=np.int32)  # per stream, of the last write(): code | detail << 8
        self._cap = np.full(n, 65536, dtype=np.int64)

    def write(self, buffers):
        """SetInput(buffers[i]) on every stream (an empty buffer is no call), then decode every stream as far as its input
        goes.  A stream's data error is reported in status and errors(), not raised; input behind the end of a finished
        stream makes its status E_STATE and raises InvalidOperationException after the other streams have gone on."""
        if len(buffers) != self.n:
            raise ValueError("one buffer per stream")
        ins = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8)) for b in buffers]
        lens = np.array([a.size for a in ins], dtype=np.int64)
        rc = _lib.lib().b200z_inflate_streams_write(self._h, _ptr_array(ins), lens.ctypes.data, self.status.ctypes.data)
        codes = self.status & 0xFF
        if rc != _lib.OK and (rc == _lib.E_STATE or not (codes == rc).any()):
            _lib.raise_for(rc)  # a failure of the call, or input for a finished stream

    def read(self):
        """everything each stream has decoded since the last read(), as a list of bytes"""
        parts = [[] for _ in range(self.n)]
        want = np.ones(self.n, dtype=bool)
        got = np.zeros(self.n, dtype=np.int64)
        while want.any():
            cap = np.where(want, self._cap, 0).astype(np.int64)
            outs = [np.empty(int(c), dtype=np.uint8) for c in cap]
            _lib.raise_for(_lib.lib().b200z_inflate_streams_read(self._h, _ptr_array(outs), cap.ctypes.data, got.ctypes.data))
            for i in np.nonzero(want)[0]:
                parts[i].append(outs[i][:got[i]].tobytes())
            want &= got == cap
            self._cap = np.where(want, np.minimum(self._cap * 4, 64 << 20), self._cap)
        return [b"".join(p) for p in parts]

    def state(self):
        """per stream: {"finished", "needs_dictionary", "total_in", "total_out", "remaining", "status"}"""
        fl = np.zeros(self.n, dtype=np.int32)
        ti, to, rem = (np.zeros(self.n, dtype=np.int64) for _ in range(3))
        st = np.zeros(self.n, dtype=np.int32)
        _lib.raise_for(_lib.lib().b200z_inflate_streams_state(self._h, fl.ctypes.data, ti.ctypes.data, to.ctypes.data,
                                                               rem.ctypes.data, st.ctypes.data))
        return [{"finished": bool(fl[i] & 1), "needs_dictionary": bool(fl[i] & 2), "total_in": int(ti[i]),
                 "total_out": int(to[i]), "remaining": int(rem[i]), "status": int(st[i])} for i in range(self.n)]

    def checks(self):
        """per stream: Inflater.Adler (WRAP_ZLIB) or the CRC-32 (WRAP_RAW_CRC32) of the output decoded so far; 0 for raw"""
        v = np.zeros(self.n, dtype=np.uint32)
        _lib.raise_for(_lib.lib().b200z_inflate_streams_check(self._h, v.ctypes.data))
        return [int(x) for x in v]

    def errors(self):
        """per stream: None, or the reference's exception message for the stream's data error"""
        out = []
        for s in self.state():
            code = s["status"] & 0xFF
            out.append(None if code in (_lib.OK, _lib.E_NEED_INPUT) else
                       _lib.lib().b200z_inflate_detail_message(s["status"]).decode())
        return out

    def set_dictionary(self, i, data):
        """Inflater.SetDictionary on stream i; the next write() decodes what waited behind the header"""
        a = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8))
        _lib.raise_for(_lib.lib().b200z_inflate_streams_set_dictionary(self._h, i, a.ctypes.data if a.size else None, a.size))

    def stats(self):
        """{"runs": stream runs, "plans": plans run, "created": plans created, "held": most compressed bytes one stream
        held at once, "workspace": most device workspace one plan took, "uploaded": host-to-device bytes of the runs}"""
        v = np.zeros(6, dtype=np.int64)
        _lib.raise_for(_lib.lib().b200z_inflate_streams_stats(self._h, v.ctypes.data, 6))
        return dict(zip(("runs", "plans", "created", "held", "workspace", "uploaded"), (int(x) for x in v)))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().b200z_inflate_streams_destroy(h)
            except Exception:  # interpreter shutdown: the module globals may already be gone
                pass

    __del__ = close

def deflate_batch(buffers, level=6, strategy=0, wrap=_lib.WRAP_RAW, end_mode=_lib.END_FINISH, devices=None):
    """Host buffers in, list of compressed bytes out (b200z_deflate_batch: H2D, kernels, D2H inside the call).
    devices: a list of CUDA device indices -- the batch is cut by bytes and every range runs on its own GPU at the same
    time (b200z_deflate_batch_multi, one host process for several GPUs).  Returns (outputs, checks)."""
    n = len(buffers)
    ins = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8)) for b in buffers]
    lens = np.array([a.size for a in ins], dtype=np.int64)
    caps = np.array([_lib.lib().b200z_deflate_bound(int(l)) + 16 for l in lens], dtype=np.int64)
    outs = [np.empty(int(c), dtype=np.uint8) for c in caps]
    out_len = np.zeros(n, dtype=np.int64)
    check = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    if devices is not None:
        dv = np.ascontiguousarray(devices, dtype=np.int32)
        rc = _lib.lib().b200z_deflate_batch_multi(dv.ctypes.data, dv.size, _ptr_array(ins), lens.ctypes.data, n, level, strategy, wrap,
                                                  end_mode, _ptr_array(outs), caps.ctypes.data, out_len.ctypes.data,
                                                  check.ctypes.data, status.ctypes.data)
    else:
        rc = _lib.lib().b200z_deflate_batch(_ptr_array(ins), lens.ctypes.data, n, level, strategy, wrap, end_mode,
                                            _ptr_array(outs), caps.ctypes.data, out_len.ctypes.data, check.ctypes.data,
                                            status.ctypes.data)
    _lib.raise_for(rc)
    return [outs[i][:out_len[i]].tobytes() for i in range(n)], check


def inflate_batch(buffers, out_caps, raise_on_error=True, wrap=_lib.WRAP_RAW, return_checks=False, devices=None):
    """Host buffers in, (outputs, in_used, status) out.  status[i] = code | detail << 8.  wrap: WRAP_RAW (raw deflate),
    WRAP_ZLIB / WRAP_GZIP (header parsed, output checksum compared with the trailer on the device; gzip: one member,
    in_used says where the next one starts), WRAP_RAW_CRC32 (raw deflate, CRC-32 of the output reported: zip entries).
    return_checks: also return the checksums of the outputs."""
    n = len(buffers)
    ins = [np.ascontiguousarray(np.frombuffer(b, dtype=np.uint8)) for b in buffers]
    lens = np.array([a.size for a in ins], dtype=np.int64)
    caps = np.ascontiguousarray(out_caps, dtype=np.int64)
    outs = [np.empty(int(c) + 1, dtype=np.uint8) for c in caps]
    out_len = np.zeros(n, dtype=np.int64)
    in_used = np.zeros(n, dtype=np.int64)
    check = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    if devices is not None:  # one host process, several GPUs (b200z_inflate_batch_multi)
        dv = np.ascontiguousarray(devices, dtype=np.int32)
        rc = _lib.lib().b200z_inflate_batch_multi(dv.ctypes.data, dv.size, _ptr_array(ins), lens.ctypes.data, n, wrap, _ptr_array(outs),
                                                  caps.ctypes.data, out_len.ctypes.data, in_used.ctypes.data, check.ctypes.data,
                                                  status.ctypes.data)
    else:
        rc = _lib.lib().b200z_inflate_batch(_ptr_array(ins), lens.ctypes.data, n, wrap, _ptr_array(outs),
                                            caps.ctypes.data, out_len.ctypes.data, in_used.ctypes.data, check.ctypes.data,
                                            status.ctypes.data)
    if raise_on_error:
        _lib.raise_for(rc)
    elif rc in (_lib.E_CUDA, _lib.E_ARG):
        _lib.raise_for(rc)
    res = [outs[i][:out_len[i]].tobytes() for i in range(n)]
    if return_checks:
        return res, in_used, status, check
    return res, in_used, status


def zip_entries(buffers, level=6):
    """Compresses the payloads of many zip entries in one device batch.  Returns, per entry, what the reference's
    ZipOutputStream.PutNextPassthroughEntry (Zip/ZipOutputStream.cs:283-333) asks for: the raw deflate stream, the CRC-32
    and the size of the uncompressed bytes (CompressedSize is len(raw)) -- the container itself (local headers, central
    directory, Zip64, name encoding) stays with the reference's own ZipOutputStream."""
    outs, checks = deflate_batch(buffers, level=level, wrap=_lib.WRAP_RAW_CRC32)
    return [{"raw": o, "crc": int(c), "size": len(b)} for o, c, b in zip(outs, checks, buffers)]


def unzip_entries(raw_streams, sizes, crcs=None):
    """The read side (ZipFile.GetInputStream + the CRC test of ZipFile.TestArchive / ZipInputStream): inflates raw entry
    streams in one device batch, CRC-32 of every output computed on the device; raises on a mismatch with `crcs`."""
    outs, used, status, checks = inflate_batch(raw_streams, sizes, wrap=_lib.WRAP_RAW_CRC32, return_checks=True)
    if crcs is not None:
        for i, (got, want) in enumerate(zip(checks, crcs)):
            if int(got) != int(want) & 0xFFFFFFFF:
                raise _lib.SharpZipBaseException("CRC mismatch in entry %d" % i)
    return outs
