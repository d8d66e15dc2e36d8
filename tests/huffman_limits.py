"""Inputs that drive DEFLATE's Huffman length limits, and a small pure-Python DEFLATE parser to check what an encoder made
of them.  Shared by tests/test_huffman_limits.py (CPU tier) and tests/test_gpu_huffman_limits.py (GPU tier).

An optimal Huffman tree for Fibonacci counts is a chain: n + 1 leaves give a code n bits deep.  DEFLATE allows 15 bits
(7 for the code-length code), so a chain of 16 or more leaves makes the encoder shorten the tree (the `overflow` repair
of `build_tree` in b200z_core.cuh), and the decoder then meets 15-bit codes, which go past its root tables."""
import heapq
import random
import zlib

import numpy as np

from sharpziplib_b200 import datagen


# ---- the reference: a plain DEFLATE parser ----------------------------------------------------------------------------
class _Bits:
    def __init__(self, data):
        self.data = bytes(data) + bytes(4)
        self.n = 8 * len(data)
        self.pos = 0

    def get(self, k):
        if self.pos + k > self.n:
            raise EOFError("stream ends inside a block")
        p = self.pos
        v = int.from_bytes(self.data[p >> 3:(p >> 3) + 4], "little") >> (p & 7)
        self.pos = p + k
        return v & ((1 << k) - 1)


def _canonical(lengths):
    """{(length, code): symbol} for the canonical code of `lengths` (RFC 1951 3.2.2)"""
    bl_count = [0] * 16
    for L in lengths:
        bl_count[L] += 1
    bl_count[0] = 0
    code, nxt = 0, [0] * 16
    for L in range(1, 16):
        code = (code + bl_count[L - 1]) << 1
        nxt[L] = code
    table = {}
    for s, L in enumerate(lengths):
        if L:
            table[(L, nxt[L])] = s
            nxt[L] += 1
    return table


def _decode(br, table):
    code = 0
    for L in range(1, 16):
        code = (code << 1) | br.get(1)
        s = table.get((L, code))
        if s is not None:
            return s
    raise ValueError("no code matches the next 15 bits")


_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
          8193, 12289, 16385, 24577]
_DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
_CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
_STATIC_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


def parse(stream, dictionary=b""):
    """Parses a raw DEFLATE stream.  Returns (blocks, bytes, bits used).  Every block is a dict with `type` (0 stored,
    1 static, 2 dynamic), `final`, and for dynamic blocks the code lengths `lit`, `dist`, `cl` and the counts of every
    symbol sent with them: `lit_counts`, `dist_counts`, `cl_counts`."""
    br = _Bits(stream)
    out = bytearray(dictionary)
    blocks = []
    while True:
        final, btype = br.get(1), br.get(2)
        blk = {"type": btype, "final": final, "start": len(out)}
        if btype == 0:
            br.pos = (br.pos + 7) & ~7
            n, nn = br.get(16), br.get(16)
            assert n ^ nn == 0xFFFF
            for _ in range(n):
                out.append(br.get(8))
        elif btype in (1, 2):
            if btype == 1:
                lit, dist = _STATIC_LIT, [5] * 30
            else:
                hlit, hdist, hclen = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                cl = [0] * 19
                for i in range(hclen):
                    cl[_CL_ORDER[i]] = br.get(3)
                ct = _canonical(cl)
                cl_counts = [0] * 19
                lens = []
                while len(lens) < hlit + hdist:
                    s = _decode(br, ct)
                    cl_counts[s] += 1
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.get(2))
                    elif s == 17:
                        lens += [0] * (3 + br.get(3))
                    else:
                        lens += [0] * (11 + br.get(7))
                assert len(lens) == hlit + hdist, "code-length run crosses the end of the lengths"
                lit, dist = lens[:hlit], lens[hlit:]
                blk.update(cl=cl, cl_counts=cl_counts)
            lt, dt = _canonical(lit), _canonical(dist)
            lit_counts, dist_counts = [0] * len(lit), [0] * len(dist)
            while True:
                s = _decode(br, lt)
                lit_counts[s] += 1
                if s < 256:
                    out.append(s)
                elif s == 256:
                    break
                else:
                    length = _LBASE[s - 257] + br.get(_LEXT[s - 257])
                    d = _decode(br, dt)
                    dist_counts[d] += 1
                    distance = _DBASE[d] + br.get(_DEXT[d])
                    assert distance <= len(out), "distance reaches in front of the stream"
                    for _ in range(length):
                        out.append(out[-distance])
            blk.update(lit=lit, dist=dist, lit_counts=lit_counts, dist_counts=dist_counts)
        else:
            raise ValueError("reserved block type 3")
        blocks.append(blk)
        if final:
            return blocks, bytes(out[len(dictionary):]), br.pos


def optimal_cost(counts):
    """sum of count * length of an optimal (unlimited) Huffman code: the sum of the weights of all merges, which is the
    same whatever order ties are taken in"""
    h = [c for c in counts if c]
    if len(h) < 2:
        return sum(h)
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        s = heapq.heappop(h) + heapq.heappop(h)
        cost += s
        heapq.heappush(h, s)
    return cost


def code_cost(lengths, counts):
    return sum(L * c for L, c in zip(lengths, counts))


def kraft(lengths):
    """the Kraft sum of a code in units of 2^-15 (32768 is a complete code)"""
    return sum(1 << (15 - L) for L in lengths if L)


def limited_trees(blocks):
    """[(block index, tree name)] for every dynamic-block tree whose emitted code costs more than an optimal Huffman code for
    its own counts: the encoder had to shorten it to meet the 15-bit (7-bit) limit"""
    found = []
    for i, b in enumerate(blocks):
        if b["type"] != 2:
            continue
        for name in ("lit", "dist", "cl"):
            if code_cost(b[name], b[name + "_counts"]) > optimal_cost(b[name + "_counts"]):
                found.append((i, name))
    return found


def check_stream(stream, data, want_limited):
    """(a)-(d) on one raw DEFLATE stream of `data`: lengths within the limits and a Kraft sum of at most 1 for every tree,
    each (block, tree) in `want_limited` costs more than optimal (the length-limit repair ran) and has a code of exactly the
    limit, and the stream decodes to `data` here and in zlib.  Returns the parsed blocks."""
    blocks, got, _ = parse(stream)
    for b in blocks:
        if b["type"] != 2:
            continue
        for name, limit in (("lit", 15), ("dist", 15), ("cl", 7)):
            assert max(b[name]) <= limit, name
            assert kraft(b[name]) <= 32768, name
    limited = limited_trees(blocks)
    for i, name in want_limited:
        assert (i, name) in limited, ("the length-limit repair did not run", i, name, limited)
        assert max(blocks[i][name]) == (7 if name == "cl" else 15), (i, name)
    assert got == data
    assert zlib.decompress(stream, -15) == data
    return blocks


# ---- designed inputs -------------------------------------------------------------------------------------------------
def fib_counts(n):
    """1, 2, 3, 5, 8, ... F(n + 1): with one more leaf of count 1 (end of block) a pure chain n bits deep"""
    out, a, b = [], 1, 2
    for _ in range(n):
        out.append(a)
        a, b = b, a + b
    return out


HUFFMAN_ONLY = 2
BLOCK_SYMBOLS = 16384   # the encoder ends a block after this many symbols (DeflaterHuffman.BUFSIZE)


def literal_chain(n, seed=0, rare_last=False, block=False):
    """n distinct byte values with the counts fib_counts(n), shuffled: under HUFFMAN_ONLY one block whose optimal literal
    tree is n deep (n >= 16: repaired to 15 bits).  rare_last: the values with the longest codes go last, so that the
    stream's tail is made of them.  block: padded to one whole block with a run of one more value, which keeps the chain
    (the run's count is larger than all the others together and joins at the root), so that what follows starts a block
    of its own."""
    rnd = random.Random(seed * 1000 + n)
    values = rnd.sample(range(256), n + 1)
    seq = []
    for v, c in zip(values, fib_counts(n)):
        seq += [v] * c
    rnd.shuffle(seq)
    if rare_last:
        rank = {v: c for v, c in zip(values, fib_counts(n))}
        seq.sort(key=lambda v: -min(rank[v], 6))
    if block:
        seq += [values[n]] * (BLOCK_SYMBOLS - len(seq))
    return bytes(seq)


def code_length_skew():
    """a natural input whose code-length code needs the 7-bit repair at levels 5-9 (a single block)"""
    return datagen.silesia_mix(3, 3000, config=9).tobytes()


# (name, input, strategy, levels, trees of block 0 that must have been shortened)
def designed():
    out = [("literal_chain_15", literal_chain(15), HUFFMAN_ONLY, range(1, 10), [])]   # exactly 15 deep: no repair
    for n in (16, 17, 18):
        out.append(("literal_chain_%d" % n, literal_chain(n), HUFFMAN_ONLY, range(1, 10), ["lit"]))
    out.append(("distance_chain_17", distance_chain(17), 0, range(1, 10), ["dist"]))
    out.append(("code_length_skew", code_length_skew(), 0, range(5, 10), ["cl"]))
    return out


def text(n, seed=3):
    return datagen.gen_text(n, seed).tobytes()


def distance_chain(ncodes=17, seed=0):
    """Random bytes, then 3-byte copies separated by one or two fresh literals, where distance code k (k < ncodes) is used
    exactly as often as the k-th count of [1] + fib_counts(ncodes - 1), in random order.  At levels 1-9 with the default
    strategy the encoder must take exactly these copies, so the block's optimal distance tree is ncodes - 1 deep.

    The bytes are picked so that no other parse is possible: every 3-byte string in the input occurs once, except where a
    copy starts; there the string's nearest earlier occurrence is the copy's source, and no earlier occurrence of it
    continues into the byte behind the copy.  So the longest match at a copy is the copy itself, at its own distance,
    and there is no match anywhere else."""
    rnd = random.Random(0xD157 + 31 * seed + ncodes)
    dists = []
    for k, c in enumerate([1] + fib_counts(ncodes - 1)):
        dists += [k] * c
    rnd.shuffle(dists)
    data = bytearray()
    seen = {}                                   # 3-byte string -> every position it starts at

    def tri(p):
        return bytes(data[p:p + 3])

    def fresh(p):
        return tri(p) not in seen

    while len(data) < 2 * _DBASE[ncodes - 1] + 64:   # a prefix in which every 3-byte string is new
        data.append(rnd.randrange(256))
        if len(data) >= 3:
            if fresh(len(data) - 3):
                seen[tri(len(data) - 3)] = [len(data) - 3]
            else:
                data.pop()
    prev = None                                 # the previous copy's start and the occurrences its string had
    for k in dists:
        lo, ext = _DBASE[k], _DEXT[k]
        for _attempt in range(1000):
            start = len(data)
            nsep = rnd.choice((1, 2))
            data += bytes(rnd.randrange(256) for _ in range(nsep))
            p = len(data)
            d = lo + rnd.randrange(1 << ext)
            for i in range(3):
                data.append(data[p - d + i])
            new = [tri(q) for q in range(max(start - 2, 0), p)]
            ok = len(set(new)) == len(new) and all(t not in seen for t in new)
            occ = seen.get(tri(p), []) + [q for q in range(max(start - 2, 0), p) if tri(q) == tri(p)]
            ok = ok and bool(occ) and max(occ) == p - d
            # the previous copy must not extend: no source of its string continues into the byte behind it
            if ok and prev is not None:
                ok = all(data[q + 3] != data[prev[0] + 3] for q in prev[1])
            if ok:
                break
            del data[start:]
        else:
            raise RuntimeError("distance_chain: no separator fits")
        for q in range(max(start - 2, 0), p):
            seen[tri(q)] = [q]
        prev = (p, occ)
        seen[tri(p)].append(p)
    data.append(rnd.randrange(256))
    while any(data[-1] == data[q + 3] for q in prev[1]):
        data[-1] = rnd.randrange(256)
    return bytes(data)
