"""GPU tier: resuming a stream inside a Huffman block.  Plans report where a stream that ran out of input can go on
(b200z_plan_get_resume_points) and can enter a block in its middle through a copy of its header
(b200z_inflate_plan_set_resume); the Inflater handle uses both, so a stream that is one huge block is read in linear time
and bounded memory whatever the SetInput granularity.  The streams are built here, token by token, and checked with
zlib and the oracle's Inflater before they are used."""
import bisect
import io
import os
import zlib

import numpy as np
import pytest

import huffman_limits as hl
from sharpziplib_b200 import datagen

pytestmark = pytest.mark.gpu

NEED_INPUT = 8
E_ARG = 1


# ---- stream builders ---------------------------------------------------------------------------------------------------
def _rev(code, n):
    return int(format(code, "0%db" % n)[::-1], 2) if n else 0


class _Bits:
    """DEFLATE bit writer: (value, bit count) pairs, packed LSB first at the end"""

    def __init__(self):
        self.v, self.n, self.pos = [], [], 0

    def put(self, val, nb):
        if nb:
            self.v.append(val)
            self.n.append(nb)
            self.pos += nb

    def align(self):
        self.put(0, (-self.pos) % 8)

    def copy(self, data, nbits):
        """the first nbits of a byte string"""
        for p in range(0, nbits, 32):
            k = min(32, nbits - p)
            self.put((int.from_bytes(data[p >> 3:(p >> 3) + 5], "little") >> (p & 7)) & ((1 << k) - 1), k)

    def bytes(self):
        n = np.array(self.n, dtype=np.int64)
        v = np.array(self.v, dtype=np.uint64)
        starts = np.repeat(np.cumsum(n) - n, n)
        within = (np.arange(starts.size, dtype=np.int64) - starts).astype(np.uint64)
        return np.packbits(((np.repeat(v, n) >> within) & 1).astype(np.uint8), bitorder="little").tobytes()


_LEN_SYM = [None] * 259  # length -> (symbol, extra bits, extra value); 258 has a code of its own (285)
for _l in range(3, 259):
    _s = 28 if _l == 258 else bisect.bisect_right(hl._LBASE[:28], _l) - 1
    _LEN_SYM[_l] = (257 + _s, hl._LEXT[_s], _l - hl._LBASE[_s])


def _dist_sym(d):
    s = bisect.bisect_right(hl._DBASE, d) - 1
    return s, hl._DEXT[s], d - hl._DBASE[s]


def _tokens(out, n_new, rng, lit_share=0.3):
    """appends about n_new bytes to `out` as literals and back-references (lengths 3..258, distances up to 32768, long
    overlapping runs included); returns the tokens: (0, byte) or (length, distance)"""
    toks = []
    end = len(out) + n_new
    while len(out) < end:
        if len(out) < 300 or rng.random() < lit_share:
            b = int(rng.integers(0, 256))
            out.append(b)
            toks.append((0, b))
            continue
        r = rng.random()
        L = 258 if r < 0.3 else int(rng.integers(3, 259))
        d = 1 if r > 0.97 else int(rng.integers(1, min(32768, len(out)) + 1))
        if d >= L:
            out += out[len(out) - d:len(out) - d + L]
        else:
            seg = out[len(out) - d:]
            out += (seg * (L // d + 1))[:L]
        toks.append((L, d))
    return toks


def _codes(lengths):
    """symbol -> (reversed code, length) of the canonical code"""
    return {s: (_rev(c, L), L) for (L, c), s in hl._canonical(lengths).items()}


def _emit(bw, toks, lit, dist, align_out=None):
    for L, v in toks:
        if L == 0:
            bw.put(*lit[v])
        else:
            s, xb, xv = _LEN_SYM[L]
            bw.put(*lit[s])
            bw.put(xv, xb)
            ds, dxb, dxv = _dist_sym(v)
            bw.put(*dist[ds])
            bw.put(dxv, dxb)
    if align_out is not None:  # static literals 144..255 take 9 bits: shift the end-of-block code to end one bit past a byte
        while (bw.pos + 6) % 8:
            bw.put(*lit[200])
            align_out.append(200)
    bw.put(*lit[256])


_STATIC_LIT = _codes(hl._STATIC_LIT)
_STATIC_DIST = _codes([5] * 30)


def _static_block(bw, out, n_new, rng, final):
    toks = _tokens(out, n_new, rng)
    bw.put(final | (1 << 1), 3)
    _emit(bw, toks, _STATIC_LIT, _STATIC_DIST, align_out=out)


def _limited_lengths(freq, limit):
    """Huffman code lengths of at most `limit` bits for the used symbols (counts flattened until the tree fits)"""
    import heapq
    f = [int(x) for x in freq]
    while True:
        heap = [(c, i, [i]) for i, c in enumerate(f) if c]
        if len(heap) == 1:
            heap.append((1, len(f), []))
        heapq.heapify(heap)
        lens = [0] * len(f)
        k = len(f) + 1
        while len(heap) > 1:
            a, b = heapq.heappop(heap), heapq.heappop(heap)
            for s in a[2] + b[2]:
                lens[s] += 1
            heapq.heappush(heap, (a[0] + b[0], k, a[2] + b[2]))
            k += 1
        if max(lens) <= limit:
            return lens
        f = [(c >> 1) | 1 if c else 0 for c in f]


def _dynamic_block(bw, out, n_new, rng, final):
    toks = _tokens(out, n_new, rng, lit_share=0.45)
    lf, df = [0] * 286, [0] * 30
    for L, v in toks:
        if L == 0:
            lf[v] += 1
        else:
            lf[_LEN_SYM[L][0]] += 1
            df[_dist_sym(v)[0]] += 1
    lf[256] += 1
    df[0] += 1
    df[29] += 1  # (two distance codes at least: a complete code)
    ll, dl = _limited_lengths(lf, 15), _limited_lengths(df, 15)
    assert hl.kraft(ll) == 32768 and hl.kraft(dl) == 32768
    while ll[-1] == 0:
        ll.pop()
    while dl[-1] == 0:
        dl.pop()
    # code lengths: runs of zeros as 17 / 18, everything else one by one
    seq, cl = [], ll + dl
    i = 0
    while i < len(cl):
        j = i
        while j < len(cl) and cl[j] == 0 and j - i < 138:
            j += 1
        if j - i >= 11:
            seq.append((18, 7, j - i - 11))
            i = j
        elif j - i >= 3:
            seq.append((17, 3, j - i - 3))
            i = j
        else:
            seq.append((cl[i], 0, 0))
            i += 1
    cf = [0] * 19
    for s, _, _ in seq:
        cf[s] += 1
    cll = _limited_lengths(cf, 7)
    cc = _codes(cll)
    hclen = 19
    while cll[hl._CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    bw.put(final | (2 << 1), 3)
    bw.put(len(ll) - 257, 5)
    bw.put(len(dl) - 1, 5)
    bw.put(max(hclen, 4) - 4, 4)
    for k in range(max(hclen, 4)):
        bw.put(cll[hl._CL_ORDER[k]], 3)
    for s, xb, xv in seq:
        bw.put(*cc[s])
        bw.put(xv, xb)
    _emit(bw, toks, _codes(ll), _codes(dl))


def _stored_block(bw, out, data, final):
    bw.put(final, 3)
    bw.align()
    bw.put(len(data), 16)
    bw.put(len(data) ^ 0xFFFF, 16)
    for b in data:
        bw.put(b, 8)
    out += data


def _not_final(comp):
    """an oracle stream with the BFINAL bit of its last block cleared, and its length in bits"""
    blocks, nbits = _scan(comp)
    c = bytearray(comp)
    h = blocks[-1]["hdr"]
    c[h >> 3] &= ~(1 << (h & 7))
    return bytes(c), nbits


def _check(oracle, comp, orig):
    assert zlib.decompress(comp, wbits=-15) == orig
    got, rem, fin = oracle.inflate(comp, max_out=len(orig) + 16)
    assert got == orig and fin and rem == 0
    return comp, orig


def build_static(oracle, n, seed=1):
    rng, out, bw = np.random.default_rng(seed), bytearray(), _Bits()
    _static_block(bw, out, n, rng, 1)
    return _check(oracle, bw.bytes(), bytes(out))


def build_dynamic(oracle, n, seed=2):
    rng, out, bw = np.random.default_rng(seed), bytearray(), _Bits()
    _dynamic_block(bw, out, n, rng, 1)
    return _check(oracle, bw.bytes(), bytes(out))


def build_mixed(oracle, n_dyn, seed=3):
    """oracle blocks, one big dynamic block, two stored blocks, a final static block"""
    rng, bw = np.random.default_rng(seed), _Bits()
    text = datagen.text_buffer(seed, 30000).tobytes()
    head, nbits = _not_final(oracle.deflate(text, level=6))
    bw.copy(head, nbits)
    out = bytearray(text)
    _dynamic_block(bw, out, n_dyn, rng, 0)
    _stored_block(bw, out, bytes(rng.integers(0, 256, 1000, dtype=np.uint8)), 0)
    _stored_block(bw, out, bytes(rng.integers(0, 256, 3000, dtype=np.uint8)), 0)
    _static_block(bw, out, 5000, rng, 1)
    return _check(oracle, bw.bytes(), bytes(out))


# ---- the pure-Python reference: where a decoder fed the first c bytes stops -----------------------------------------------
def _scan(stream):
    """blocks of a raw stream: header bit, body bit (stored: the header bit), end bit, output position, type, and for
    Huffman blocks every symbol as (first bit, bit behind it incl. extra bits, output position, dist-extra bit range)"""
    br = hl._Bits(stream)
    blocks, outn = [], 0
    while True:
        hdr = br.pos
        final, btype = br.get(1), br.get(2)
        blk = {"hdr": hdr, "type": btype, "out": outn, "syms": []}
        if btype == 0:
            br.pos = (br.pos + 7) & ~7
            n = br.get(16)
            br.get(16)
            blk["data"] = br.pos >> 3
            br.pos += 8 * n
            outn += n
            blk["body"] = hdr
        else:
            if btype == 1:
                lit, dist = hl._STATIC_LIT, [5] * 30
            else:
                hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[hl._CL_ORDER[i]] = br.get(3)
                ct = hl._canonical(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = hl._decode(br, ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.get(2))
                    elif s == 17:
                        lens += [0] * (3 + br.get(3))
                    else:
                        lens += [0] * (11 + br.get(7))
                lit, dist = lens[:hlit], lens[hlit:]
            blk["body"] = br.pos
            lt, dt = hl._canonical(lit), hl._canonical(dist)
            while True:
                p = br.pos
                s = hl._decode(br, lt)
                dx = None
                if s == 256:
                    blk["syms"].append((p, br.pos, outn, None))
                    break
                if s < 256:
                    outn += 1
                else:
                    length = hl._LBASE[s - 257] + br.get(hl._LEXT[s - 257])
                    d = hl._decode(br, dt)
                    x0 = br.pos
                    br.get(hl._DEXT[d])
                    dx = (x0, br.pos)
                    blk["syms"].append((p, br.pos, outn, dx))
                    outn += length
                    continue
                blk["syms"].append((p, br.pos, outn - 1, None))
        blk["end"] = br.pos
        blocks.append(blk)
        if final:
            return blocks, br.pos


def _expected_stop(blocks, c):
    """(hdr_bit, body_bit, sym_bit, out_pos, block out) of a decoder that has the first c bytes, or None if it ends"""
    C = 8 * c
    for b in blocks:
        if b["type"] == 0:
            if b["end"] > C:
                return b["hdr"], b["hdr"], b["hdr"], b["out"], b["out"]
            continue
        if b["body"] > C:
            return b["hdr"], b["hdr"], b["hdr"], b["out"], b["out"]
        for p, e, o, _ in b["syms"]:
            if e > C:
                return b["hdr"], b["body"], p, o, b["out"]
    return None


def _cuts(blocks):
    """byte cuts: in a header, right behind a header, in a distance's extra bits, one bit short of an end-of-block code,
    in a stored block, at a block boundary"""
    cuts = {}
    for b in blocks:
        if b["type"] == 0:
            cuts.setdefault("stored", b["data"] + 100 if b["end"] - 8 * b["data"] > 800 else b["data"] + 1)
            cuts.setdefault("boundary", b["end"] >> 3)
            continue
        if (b["body"] >> 3) > (b["hdr"] >> 3) + 1:
            cuts.setdefault("header", ((b["hdr"] + b["body"]) // 2) >> 3)
        cuts.setdefault("after_header", (b["body"] + 7) >> 3)
        for p, e, o, dx in b["syms"]:
            if dx and 8 * ((dx[0] >> 3) + 1) < dx[1]:  # a byte boundary strictly inside the distance's extra bits
                cuts.setdefault("extra", (dx[0] >> 3) + 1)
                break
        p, e = b["syms"][-1][:2]
        if e % 8 == 1:
            cuts.setdefault("eob_minus_1", e >> 3)
    return cuts


def _run(z, comps, caps, windows, start_bits, skip_bits):
    import torch
    n = len(comps)
    ip = z.InflatePlan([len(c) for c in comps], caps, dict_lens=[len(w) for w in windows])
    ip.set_resume(start_bits, skip_bits)
    hin = np.zeros(ip.in_bytes, dtype=np.uint8)
    for i in range(n):
        blob = windows[i] + comps[i]
        o = int(ip.in_offsets[i])
        hin[o:o + len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    di = torch.from_numpy(hin).cuda()
    do = torch.zeros(ip.out_bytes, dtype=torch.uint8, device="cuda")
    d_len = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_st = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_used = torch.zeros(n, dtype=torch.int64, device="cuda")
    ip.run(di, do, d_len, d_st, None, d_used)
    torch.cuda.synchronize()
    res = ip.resume_points()
    rbit, rpos = ip.restart_points()
    o2 = do.cpu().numpy()
    lens = d_len.cpu().numpy()
    outs = [o2[int(o):int(o) + int(l)].tobytes() for o, l in zip(ip.out_offsets, lens)]
    ip.close()
    return outs, d_st.cpu().numpy(), d_used.cpu().numpy(), res, (rbit, rpos)


def _small_streams(oracle):
    return [("static", *build_static(oracle, 40000)), ("dynamic", *build_dynamic(oracle, 40000)),
            ("mixed", *build_mixed(oracle, 20000))]


@pytest.mark.parametrize("mode", ["pipeline", "serial"])
def test_plan_resume_points_and_mid_block_entry(z, oracle, mode):
    """Streams cut at chosen bytes report the resume point the parser predicts; a second plan entered there through the
    window image and a copy of the block header produces exactly the rest"""
    if mode == "serial":
        os.environ["B200Z_INFLATE"] = "serial"  # read when a plan is built
    try:
        cases = []
        for name, comp, orig in _small_streams(oracle):
            blocks, _ = _scan(comp)
            cuts = _cuts(blocks)
            want = {"static": {"after_header", "extra", "eob_minus_1"}, "dynamic": {"header", "after_header", "extra"},
                    "mixed": {"header", "after_header", "extra", "eob_minus_1", "stored", "boundary"}}[name]
            assert want <= set(cuts), (name, cuts)
            for kind, c in sorted(cuts.items()):
                cases.append((name, kind, comp, orig, c, _expected_stop(blocks, c)))
        n = len(cases)
        outs, st, used, (hb, bb, sb, so), (rbit, rpos) = _run(
            z, [c[:cut] for _, _, c, _, cut, _ in cases], [len(o) + 64 for _, _, _, o, _, _ in cases], [b""] * n, [0] * n, [0] * n)
        second = []
        for i, (name, kind, comp, orig, cut, exp) in enumerate(cases):
            h, b, s, o, blk_out = exp
            assert int(st[i]) == NEED_INPUT, (name, kind, st[i])
            assert (int(hb[i]), int(bb[i]), int(sb[i]), int(so[i])) == (h, b, s, o), (name, kind, cut, exp)
            assert (int(rbit[i]), int(rpos[i])) == (h, blk_out), (name, kind)  # the restart point keeps its meaning
            assert outs[i] == orig[:o], (name, kind)
            if s != h:  # inside the block: header copy + tail from the symbol's byte
                hdr = comp[h >> 3:(b + 7) >> 3]
                second.append((hdr + comp[s >> 3:], h & 7, 8 * len(hdr) + (s & 7), len(hdr), s >> 3))
            else:
                second.append((comp[h >> 3:], h & 7, 0, 0, h >> 3))
        assert sum(1 for name, kind, *_ in cases if kind in ("extra", "eob_minus_1", "after_header")) >= 6
        outs2, st2, used2, _, _ = _run(z, [x[0] for x in second], [len(o) + 64 for _, _, _, o, _, _ in cases],
                                       [orig[max(0, e[3] - 32768):e[3]] for _, _, _, orig, _, e in cases],
                                       [x[1] for x in second], [x[2] for x in second])
        for i, (name, kind, comp, orig, cut, exp) in enumerate(cases):
            _, _, _, H, tail = second[i]
            assert int(st2[i]) == 0, (name, kind, st2[i])
            assert outs[i] + outs2[i] == orig, (name, kind)
            assert tail + int(used2[i]) - H == len(comp), (name, kind)  # RemainingInput stays exact
    finally:
        os.environ.pop("B200Z_INFLATE", None)


@pytest.mark.parametrize("mode", ["pipeline", "serial"])
def test_plan_mid_block_entry_is_refused_for_stored_blocks_and_inside_headers(z, oracle, mode):
    if mode == "serial":
        os.environ["B200Z_INFLATE"] = "serial"
    try:
        comp, orig = build_dynamic(oracle, 3000)
        blocks, _ = _scan(comp)
        body = blocks[0]["body"]
        stored = zlib.compressobj(0, zlib.DEFLATED, -15)
        sc = stored.compress(b"abc" * 100) + stored.flush()
        outs, st, _, _, _ = _run(z, [comp, sc, comp], [len(orig) + 64, 400, len(orig) + 64], [b""] * 3, [0, 0, 0],
                                 [body - 1, 40, body])
        assert [int(x) & 0xFF for x in st] == [E_ARG, E_ARG, 0]
        assert outs[2] == orig  # (a jump to the header's end is no jump at all)
    finally:
        os.environ.pop("B200Z_INFLATE", None)


# ---- the Inflater handle ------------------------------------------------------------------------------------------------
def _feed(z, comp, chunk, nowrap=True, out_chunk=1 << 16):
    inf = z.Inflater(nowrap)
    buf = bytearray(out_chunk)
    got = bytearray()
    pos = 0
    while not inf.IsFinished:
        n = inf.Inflate(buf)
        got += buf[:n]
        if n == 0 and inf.IsNeedingInput and not inf.IsFinished:
            if pos >= len(comp):
                raise EOFError("Unexpected EOF")
            inf.SetInput(comp[pos:pos + chunk])
            pos += chunk
    return bytes(got), inf, pos


def _whole(z, comp, nowrap=True):
    got, inf, pos = _feed(z, comp, len(comp), nowrap)
    return got, inf.TotalIn, inf.TotalOut, inf.RemainingInput


# bounds the handle keeps (DESIGN.md 7a): compressed bytes held <= largest SetInput + K_HELD_COMP, output bytes held <= the
# output of one run (at most 1032 bytes per input byte) + the window, and no byte is decoded twice
K_HELD_COMP = 65540 + 600
K_HELD_OUT = 32768


def _check_feed(z, name, comp, orig, chunk, nowrap=True):
    got, inf, pos = _feed(z, comp + b"TAIL", chunk, nowrap)
    assert got == orig, (name, chunk)
    fed = min(pos, len(comp) + 4)
    assert inf.IsFinished and inf.TotalOut == len(orig) and inf.TotalIn == len(comp), (name, chunk)
    assert inf.RemainingInput == fed - len(comp), (name, chunk)
    s = inf.stats()
    assert s["decoded"] == inf.TotalOut, (name, chunk, s)
    assert s["max_comp_held"] <= chunk + K_HELD_COMP, (name, chunk, s)
    assert s["max_out_held"] <= 1032 * (chunk + K_HELD_COMP) + K_HELD_OUT, (name, chunk, s)
    return s


@pytest.fixture(scope="module")
def big(oracle):
    return {"static64": build_static(oracle, 64 << 20, seed=11), "dynamic16": build_dynamic(oracle, 16 << 20, seed=12),
            "mixed": build_mixed(oracle, 4 << 20, seed=13)}


def test_handle_one_huge_block_at_any_granularity(z, oracle, big):
    for name, (comp, orig) in big.items():
        for chunk in (4096, 4093, 1 << 20):
            s = _check_feed(z, name, comp, orig, chunk)
            if name != "mixed":  # (no stored block to wait for: a header or a symbol is all that is kept)
                assert s["max_comp_held"] <= chunk + 1024, (name, chunk, s)
            if chunk < 8192:  # nothing close to the block (4, 16, 64 MiB) is held
                assert s["max_out_held"] < 1 << 20, (name, chunk, s)


def test_handle_small_streams_odd_and_byte_feeds(z, oracle):
    for name, comp, orig in _small_streams(oracle):
        for chunk in (7, 4093):
            _check_feed(z, name, comp, orig, chunk)
    comp, orig = build_static(oracle, 3000, seed=5)
    _check_feed(z, "static_small", comp, orig, 1)


def test_handle_restart_streams(z, oracle):
    import test_gpu_restart
    for name, orig, comp in test_gpu_restart._streams(oracle):
        for chunk in (7, 4096, 4093, 1 << 20):
            if chunk == 7 and len(comp) > 100000:
                continue  # (seven bytes a call over the long ones costs minutes of round trips, nothing more)
            _check_feed(z, name, comp, orig, chunk)


def test_zlib_trailer_in_pieces_decodes_the_final_block_once(z, big):
    comp, orig = big["dynamic16"]
    zc = b"\x78\x9c" + comp + zlib.adler32(orig).to_bytes(4, "big")
    assert zlib.decompress(zc) == orig
    inf = z.Inflater(False)
    buf = bytearray(1 << 20)
    got = bytearray()
    inf.SetInput(zc[:-4])
    while True:
        n = inf.Inflate(buf)
        if n == 0:
            break
        got += buf[:n]
    runs = inf.stats()["runs"]
    for k in range(4):
        assert not inf.IsFinished and inf.IsNeedingInput
        inf.SetInput(zc[len(zc) - 4 + k:len(zc) - 3 + k])
        n = inf.Inflate(buf)
        got += buf[:n]
    assert inf.IsFinished and bytes(got) == orig and inf.Adler == zlib.adler32(orig)
    s = inf.stats()
    assert s["runs"] == runs and s["decoded"] == len(orig), s


def test_inflater_input_stream_reads_the_64_mib_block(z, big):
    comp, orig = big["static64"]
    ins = z.InflaterInputStream(io.BytesIO(comp), z.Inflater(True))
    assert ins.read() == orig
