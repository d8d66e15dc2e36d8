"""GPU tier: Inflater sets (b200z_inflate_streams_*, InflaterSet).  Every stream is compared with the oracle's Inflater and
with an Inflater handle fed the same SetInput pieces: output (in mid-stream a prefix of the reference's, as the handle's
is), IsFinished and IsNeedingDictionary after every write, TotalIn, TotalOut, RemainingInput and Adler / CRC-32 once the
stream has finished, and the error message.  Tests named *small* also run on the CUDA emulator (tests/test_inflate_streams_emu.py), which builds the library
with small plan bounds, so that the same writes split into several plans there."""
import random
import zlib

import numpy as np
import pytest

from sharpziplib_b200 import _lib, datagen

pytestmark = pytest.mark.gpu

WRAPS = [_lib.WRAP_RAW, _lib.WRAP_ZLIB, _lib.WRAP_RAW_CRC32]


def _drain(inflate, needs_input, finished, needs_dict):
    out = bytearray()
    for _ in range(1 << 20):
        b = inflate()
        out += b
        if not b and (needs_input() or finished() or needs_dict()):
            return bytes(out)
    raise AssertionError("no progress")


class Reference:
    """one stream as the reference reads it: the oracle's Inflater, SetInput per piece, Inflate until it needs input"""

    def __init__(self, oracle, wrap, dictionary=None):
        self.oracle = oracle
        self.i = oracle.Inflater(nowrap=wrap != _lib.WRAP_ZLIB)
        self.dictionary = dictionary
        self.out = bytearray()
        self.error = None
        self.late = False

    def write(self, piece):
        if self.error is not None or not piece:
            return
        if self.i.finished:
            self.late = True
            return
        self.i.set_input(piece)
        try:
            while True:
                self.out += _drain(lambda: self.i.inflate(1 << 20), lambda: self.i.needs_input, lambda: self.i.finished,
                                   lambda: self.i.needs_dictionary)
                if not (self.i.needs_dictionary and self.dictionary is not None):
                    return
                self.i.set_dictionary(self.dictionary)
                self.dictionary = None
        except self.oracle.OracleError as e:
            self.error = e.msg


class Handle:
    """the same pieces on an Inflater handle"""

    def __init__(self, z, wrap, dictionary=None):
        self.i = z.Inflater(wrap != _lib.WRAP_ZLIB)
        self.z = z
        self.dictionary = dictionary
        self.out = bytearray()
        self.buf = bytearray(1 << 20)
        self.error = None

    def write(self, piece):
        if self.error is not None or not piece or self.i.IsFinished:
            return
        self.i.SetInput(piece)
        try:
            while True:
                self.out += _drain(lambda: bytes(self.buf[:self.i.Inflate(self.buf)]), lambda: self.i.IsNeedingInput,
                                   lambda: self.i.IsFinished, lambda: self.i.IsNeedingDictionary)
                if not (self.i.IsNeedingDictionary and self.dictionary is not None):
                    return
                self.i.SetDictionary(self.dictionary)
                self.dictionary = None
        except self.z.SharpZipBaseException as e:
            self.error = str(e)


def _pieces(comp, size, rng):
    """comp cut into pieces of `size` bytes (0: random sizes of 1..9000)"""
    out, p = [], 0
    while p < len(comp):
        n = size or rng.randint(1, 9000)
        out.append(comp[p:p + n])
        p += n
    return out


def run_set(z, oracle, wrap, streams, sizes, dictionaries=None, handles=True, seed=0):
    """streams[i] = (compressed, original or None); sizes[i] = piece size of stream i (0: mixed), or its list of pieces.
    Writes round by round (streams whose pieces ran out get empty writes) and checks every stream after every write;
    returns the set."""
    rng = random.Random(seed)
    n = len(streams)
    dictionaries = dictionaries or [None] * n
    pieces = [sizes[i] if isinstance(sizes[i], list) else _pieces(c, sizes[i], rng) for i, (c, _) in enumerate(streams)]
    refs = [Reference(oracle, wrap, dictionaries[i]) for i in range(n)]
    hs = [Handle(z, wrap, dictionaries[i]) for i in range(n)] if handles else None
    s = z.InflaterSet(n, wrap)
    got = [bytearray() for _ in range(n)]
    for r in range(max(len(p) for p in pieces) + 1):
        bufs = [p[r] if r < len(p) else b"" for p in pieces]
        for i in range(n):
            refs[i].write(bufs[i])
            if hs:
                hs[i].write(bufs[i])
        try:
            s.write(bufs)
        except z.InvalidOperationException:
            pass
        for i, b in enumerate(s.read()):
            got[i] += b
        waiting = [i for i, st in enumerate(s.state()) if st["needs_dictionary"] and dictionaries[i] is not None]
        for i in waiting:
            s.set_dictionary(i, dictionaries[i])
            dictionaries[i] = None
        if waiting:  # (the next write decodes what waited behind the header)
            s.write([b""] * n)
            for i, b in enumerate(s.read()):
                got[i] += b
        st, ck = s.state(), s.checks()
        for i in range(n):
            ref = refs[i]
            code = s.status[i] & 0xFF
            if ref.late:
                assert code == _lib.E_STATE, (i, r)
                ref.late = False
            if ref.error is not None:
                msg = s.errors()[i]
                assert msg and msg in ref.error, (i, msg, ref.error)
                k = min(len(got[i]), len(ref.out))  # (what both delivered in front of it)
                assert bytes(got[i][:k]) == bytes(ref.out[:k]), i
                continue
            # in mid-stream the set's output may lag behind the reference's, as the handle's does (a stored block comes
            # out once it is complete); the handle fed the same pieces has exactly the same
            assert bytes(ref.out).startswith(bytes(got[i])), (i, r, len(got[i]), len(ref.out))
            if hs:
                assert bytes(hs[i].out) == bytes(got[i]), (i, r)
            assert st[i]["total_out"] == len(got[i]), (i, r)
            assert st[i]["finished"] == ref.i.finished, (i, r)
            assert st[i]["needs_dictionary"] == ref.i.needs_dictionary, (i, r)
            if ref.i.finished:
                assert bytes(got[i]) == bytes(ref.out), (i, r)
                assert st[i]["total_in"] == ref.i.total_in, (i, r)
                assert st[i]["remaining"] == ref.i.remaining_input, (i, r)
                assert st[i]["total_out"] == ref.i.total_out, (i, r)
                assert code == _lib.OK, (i, r, s.status[i])
                if wrap == _lib.WRAP_ZLIB:
                    assert ck[i] == ref.i.adler & 0xFFFFFFFF, i
                if wrap == _lib.WRAP_RAW_CRC32:
                    assert ck[i] == zlib.crc32(bytes(got[i])), i
            elif ref.i.needs_dictionary:
                assert ck[i] == ref.i.adler & 0xFFFFFFFF, i
    for i, (c, orig) in enumerate(streams):
        if orig is not None and refs[i].error is None:
            assert bytes(got[i]) == orig and s.state()[i]["finished"], i
    return s


def _data(i, n):
    return (datagen.text_buffer if i % 2 else datagen.silesia_mix)(100 + i, n).tobytes()


def _oracle_streams(oracle, wrap, count, size, levels=range(10)):
    out = []
    for i in range(count):
        d = _data(i, size + 997 * i % size if size else 0)
        lv = list(levels)[i % len(levels)]
        out.append((oracle.deflate(d, level=lv, nowrap=wrap != _lib.WRAP_ZLIB), d))
    return out


@pytest.mark.parametrize("wrap", WRAPS)
def test_small_levels_and_piece_sizes(z, oracle, wrap):
    streams = _oracle_streams(oracle, wrap, 10, 12000)
    run_set(z, oracle, wrap, streams, [517, 4093, 4096, 0, 1 << 20, 4093, 0, 4096, 1 << 20, 517])


@pytest.mark.parametrize("n", [1, 2, 37])
def test_set_sizes_finish_in_different_writes(z, oracle, n):
    streams = [(oracle.deflate(_data(i, 300 * (i % 9) + 50), level=i % 10, nowrap=False), _data(i, 300 * (i % 9) + 50))
               for i in range(n)]
    run_set(z, oracle, _lib.WRAP_ZLIB, streams, [[1, 7, 517, 0][i % 4] for i in range(n)])


def test_zlib_written_streams_and_byte_feeds(z, oracle):
    d = [_data(i, 20000) for i in range(4)]
    streams = [(zlib.compress(d[0], 9), d[0]), (zlib.compress(d[1], 1), d[1]), (zlib.compress(b"", 6), b""),
               (zlib.compress(d[3][:300], 6), d[3][:300])]
    run_set(z, oracle, _lib.WRAP_ZLIB, streams, [4093, 7, 1, 1])
    raw = [(c[2:-4], o) for c, o in streams]
    run_set(z, oracle, _lib.WRAP_RAW, raw, [4096, 1, 1, 1])


def test_small_trailing_bytes_and_trailer_bytewise(z, oracle):
    d = _data(3, 40000)
    zc = oracle.deflate(d, level=6, nowrap=False)
    rc = oracle.deflate(d, level=6, nowrap=True)
    # the trailer of stream 0 arrives one byte per write; streams 1 and 2 carry bytes behind their end
    streams = [(zc, d), (zc + b"TRAILING", None), (rc + b"BEHIND THE END", None)]
    trailer_bytewise = [zc[:-4]] + [zc[k:k + 1] for k in range(len(zc) - 4, len(zc))]
    s = run_set(z, oracle, _lib.WRAP_ZLIB, [streams[0], streams[1]], [trailer_bytewise, 4096])
    assert s.state()[1]["remaining"] == 8
    s = run_set(z, oracle, _lib.WRAP_RAW, [streams[2]], [len(streams[2][0])])
    assert s.state()[0]["remaining"] == 14
    # input after the end: E_STATE for that stream alone
    s = z.InflaterSet(2, _lib.WRAP_RAW)
    s.write([rc, rc[:100]])
    with pytest.raises(z.InvalidOperationException):
        s.write([b"more", rc[100:]])
    assert s.status[0] & 0xFF == _lib.E_STATE and s.status[1] == _lib.OK
    out = s.read()
    assert out == [d, d]


def test_cuts_inside_headers_extra_bits_and_stored_blocks(z, oracle):
    import test_gpu_inflate_resume as T
    cases = T._small_streams(oracle)
    streams = [(comp, orig) for _, comp, orig in cases]
    for size in (1, 3, 5, 11):
        run_set(z, oracle, _lib.WRAP_RAW, streams, [size] * len(streams), handles=size == 5)


def test_small_preset_dictionary(z, oracle):
    text = _data(8, 60000)
    dictionary = _data(9, 50000)  # longer than the window: only its tail matters
    co = zlib.compressobj(6, zlib.DEFLATED, 15, 9, zlib.Z_DEFAULT_STRATEGY, dictionary)
    c = co.compress(text) + co.flush()
    run_set(z, oracle, _lib.WRAP_ZLIB, [(c, text), (c, text)], [4096, 1000], dictionaries=[dictionary, dictionary])
    s = z.InflaterSet(2, _lib.WRAP_ZLIB)
    s.write([c[:4000], b""])
    st = s.state()
    assert st[0]["needs_dictionary"] and s.checks()[0] == zlib.adler32(dictionary)
    with pytest.raises(z.SharpZipBaseException, match="Wrong adler checksum"):
        s.set_dictionary(0, dictionary[1:])
    with pytest.raises(z.InvalidOperationException, match="Dictionary is not needed"):
        s.set_dictionary(1, dictionary)
    s.set_dictionary(0, dictionary)
    s.write([c[4000:], b""])
    assert s.read()[0] == text and s.state()[0]["finished"]


def test_small_corrupt_and_truncated_streams_leave_the_others_alone(z, oracle):
    streams = _oracle_streams(oracle, _lib.WRAP_ZLIB, 5, 50000, levels=[6])
    bad = bytearray(streams[1][0])
    bad[len(bad) // 3] ^= 0xFF
    hdr = bytearray(streams[3][0])
    hdr[1] ^= 1  # "Header checksum illegal"
    trunc = streams[2][0][:len(streams[2][0]) // 2]
    cases = [streams[0], (bytes(bad), None), (trunc, None), (bytes(hdr), None), streams[4]]
    s = run_set(z, oracle, _lib.WRAP_ZLIB, cases, [4096] * 5)
    st = s.state()
    assert st[0]["finished"] and st[4]["finished"]
    assert st[2]["status"] & 0xFF == _lib.E_NEED_INPUT and not st[2]["finished"]
    assert st[3]["status"] & 0xFF == _lib.E_DATA and s.errors()[3] == "Header checksum illegal"
    code = st[1]["status"] & 0xFF
    assert code == _lib.E_DATA or code == _lib.E_NEED_INPUT  # (a flipped bit may leave a stream that never ends)


def test_small_output_larger_than_its_capacity_is_decoded_once(z, oracle):
    d = bytes(700000)  # (more than the 589824 bytes of output capacity a run of its size gets first)
    c = oracle.deflate(d, level=6, nowrap=True)
    s = z.InflaterSet(2, _lib.WRAP_RAW_CRC32)
    s.write([c, c[:10]])
    s.write([b"", c[10:]])
    out = s.read()
    assert out == [d, d]
    assert s.checks() == [zlib.crc32(d)] * 2
    st = s.stats()
    # one run per capacity step of stream 0 (each goes on from its resume point), at most as many for stream 1
    assert st["runs"] <= 8, st


def test_small_plans_split_and_are_reused(z, oracle):
    n = 12
    data = [_data(i, 30000) for i in range(n)]
    comp = [oracle.deflate(d, level=6, nowrap=True) for d in data]
    s = z.InflaterSet(n, _lib.WRAP_RAW)
    got = [bytearray() for _ in range(n)]
    created = []
    for p in range(0, max(len(c) for c in comp), 4096):
        s.write([c[p:p + 4096] for c in comp])
        for i, b in enumerate(s.read()):
            got[i] += b
        if p + 4096 < min(len(c) for c in comp):  # (every stream due, with a full piece)
            created.append(s.stats()["created"])
    assert [bytes(g) for g in got] == data
    st = s.stats()
    assert st["plans"] >= st["runs"] // n  # (one plan per write at least)
    assert created[-1] == created[0], created  # equal writes: plans only in the first
    assert st["held"] <= 4096 + 65540 + 600, st
    total = sum(len(c) for c in comp)
    assert st["uploaded"] <= total + st["runs"] * 700, st


def test_many_streams_and_pieces(z, oracle):
    for n, size, piece in ((1024, 3000, 4096), (37, 2 << 20, 1 << 20), (256, 200000, 4096)):
        streams = [(oracle.deflate(_data(i, size), level=6, nowrap=True), None) for i in range(n)]
        s = run_set(z, oracle, _lib.WRAP_RAW, streams, [piece] * n, handles=n <= 37)
        st = s.stats()
        assert st["held"] <= piece + 65540 + 600, st
        if piece == 4096:
            assert st["uploaded"] <= sum(len(c) for c, _ in streams) + st["runs"] * 700, st


@pytest.fixture(scope="module")
def big(oracle):
    import test_gpu_inflate_resume as T
    return {"static64": T.build_static(oracle, 64 << 20, seed=11), "dynamic16": T.build_dynamic(oracle, 16 << 20, seed=12),
            "mixed": T.build_mixed(oracle, 4 << 20, seed=13)}


def test_huge_blocks_in_a_set(z, oracle, big):
    names = list(big)
    streams = [big[k] for k in names]
    for piece in (4096, 4093, 1 << 20):
        s = z.InflaterSet(len(streams), _lib.WRAP_RAW)
        got = [bytearray() for _ in streams]
        rounds = max(len(c) for c, _ in streams) // piece + 1
        for r in range(rounds):
            s.write([c[r * piece:(r + 1) * piece] for c, _ in streams])
            for i, b in enumerate(s.read()):
                got[i] += b
        for i, (c, orig) in enumerate(streams):
            assert bytes(got[i]) == orig, (names[i], piece)
        st = s.stats()
        assert st["held"] <= piece + 65540 + 600, (piece, st)
