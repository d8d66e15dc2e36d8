"""GPU tier: DEFLATE's Huffman length limits on the device.  The deflate kernels must give the oracle's bytes for inputs
whose trees need the length-limit repair (tests/huffman_limits.py), and both inflate kernels -- the block-parallel
pipeline and the serial kernel -- must decode streams full of 15-bit codes, whole, truncated inside them, and fed in
pieces, as the oracle's Inflater does.  Tests whose name holds "emu" are small enough for the CUDA emulator; the CPU
tier runs them there."""
import random
import zlib

import numpy as np
import pytest

import huffman_limits as H
from helpers import oracle_calls
from sharpziplib_b200 import datagen
from test_gpu_inflate_parallel import _run_plan, _serial

pytestmark = pytest.mark.gpu


def _ordinary():
    return [datagen.silesia_mix(c, 3000 + 1717 * c).tobytes() for c in range(4)] + [b"", b"x"]


def _oracle_wrap(oracle, d, level, strategy, wrap, end_mode):
    return oracle.deflate(d, level=level, nowrap=not wrap, strategy=strategy, pattern=end_mode)


# ---- deflate ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("strategy", [0, 1, 2])
def test_deflate_batch_designed_inputs(z, oracle, strategy):
    """the designed inputs in batches with ordinary streams: levels 1-9, raw and zlib framing, Finish() and Flush() then
    Finish()"""
    bufs = [d for _, d, _, _, _ in H.designed()] + _ordinary()
    for level in range(1, 10):
        for wrap in (0, 1):
            for end_mode in (0, 1):
                outs, _ = z.deflate_batch(bufs, level=level, strategy=strategy, wrap=wrap, end_mode=end_mode)
                for i, (d, o) in enumerate(zip(bufs, outs)):
                    assert o == _oracle_wrap(oracle, d, level, strategy, wrap, end_mode), (i, level, wrap, end_mode)


def test_emu_deflate_batch_repairs(z, oracle):
    """every designed input in the configuration that needs the repair, level 6: the GPU's stream reaches it too"""
    for name, d, strategy, levels, trees in H.designed():
        outs, _ = z.deflate_batch([d, _ordinary()[0]], level=6, strategy=strategy)
        assert outs[0] == oracle.deflate(d, level=6, strategy=strategy), name
        H.check_stream(outs[0], d, [(0, t) for t in trees])


def _gpu_calls(z, level, segs, strategy=0):
    d = z.Deflater(level, True)
    d.SetStrategy(strategy)
    out, buf = bytearray(), bytearray(1 << 16)

    def drain():
        while True:
            k = d.Deflate(buf)
            if k <= 0:
                return
            out.extend(buf[:k])
    for i, (seg, chunks) in enumerate(segs):
        pos = 0
        for c in chunks:
            d.SetInput(seg[pos:pos + c])
            pos += c
            drain()
        d.Flush() if i + 1 < len(segs) else d.Finish()
        drain()
    return bytes(out)


def _oracle_calls(level, segs, strategy=0):
    if strategy == 0:
        return oracle_calls(level, segs, None, True, nowrap=True)
    from oracle_lib import Deflater
    d = Deflater(level, nowrap=True)
    d.set_strategy(strategy)
    out = bytearray()

    def drain():
        while True:
            b = d.deflate(4096)
            if not b:
                return
            out.extend(b)
    for i, (seg, chunks) in enumerate(segs):
        pos = 0
        for c in chunks:
            d.set_input(seg[pos:pos + c])
            pos += c
            drain()
        d.flush() if i + 1 < len(segs) else d.finish()
        drain()
    return bytes(out)


def test_emu_deflater_handle_pieces_and_flush(z, oracle):
    """the Deflater handle: SetInput in pieces, a Flush() around the designed part (its block still needs the repair) and a
    Flush() in the middle of it"""
    chain, dist, t = H.literal_chain(17), H.distance_chain(17), H.text(9000)
    cases = [(H.HUFFMAN_ONLY, [(t[:3000], [1000, 2000]), (chain, [1, 2, 4000, len(chain) - 4003]), (t[3000:], [6000])], 1),
             (H.HUFFMAN_ONLY, [(chain[:3000], [3000]), (chain[3000:], [500, len(chain) - 3500])], None),
             (0, [(dist, [7, 10000, len(dist) - 10007]), (t, [9000])], 0),
             (0, [(dist[:9000], [9000]), (dist[9000:] + t, [len(dist) - 9000 + len(t)])], None)]
    for level in (1, 6):
        for ci, (strategy, segs, block) in enumerate(cases):
            got = _gpu_calls(z, level, segs, strategy)
            assert got == _oracle_calls(level, segs, strategy), (level, ci)
            if block is not None:
                blocks, back, _ = H.parse(got)
                assert back == b"".join(s for s, _ in segs)
                tree = "lit" if strategy else "dist"
                assert any(name == tree for _, name in H.limited_trees(blocks)), (level, ci)


def test_plan_in_two_stages(z, oracle):
    """STAGE_SEARCH then STAGE_ENCODE at level 6 on the designed inputs"""
    import torch
    for strategy in (0, H.HUFFMAN_ONLY):
        bufs = [d for _, d, _, _, _ in H.designed()] + _ordinary()[:2]
        plan = z.DeflatePlan([len(b) for b in bufs], level=6, strategy=strategy)
        blob = np.zeros(plan.in_bytes, np.uint8)
        for o, b in zip(plan.in_offsets, bufs):
            blob[o:o + len(b)] = np.frombuffer(b, np.uint8)
        d_in = torch.from_numpy(blob).cuda()
        d_out = torch.zeros(plan.out_bytes, dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(plan.n, dtype=torch.int64, device="cuda")
        d_st = torch.ones(plan.n, dtype=torch.int32, device="cuda")
        plan.run(d_in, d_out, d_len, d_st, stages=z.STAGE_SEARCH)
        plan.run(d_in, d_out, d_len, d_st, stages=z.STAGE_ENCODE)
        torch.cuda.synchronize()
        assert d_st.cpu().tolist() == [0] * plan.n
        for i, b in enumerate(bufs):
            o = int(plan.out_offsets[i])
            assert d_out[o:o + int(d_len[i])].cpu().numpy().tobytes() == oracle.deflate(b, level=6, strategy=strategy), \
                (strategy, i)
        plan.close()


# ---- inflate ------------------------------------------------------------------------------------------------------------
def _zlib_raw(d, strategy):
    co = zlib.compressobj(6, zlib.DEFLATED, -15, 8, strategy)
    return co.compress(d) + co.flush()


def _streams(oracle):
    """(input, raw DEFLATE stream) pairs: the oracle's streams of the designed inputs, and zlib's, HUFFMAN_ONLY and default
    (zlib limits lengths its own way and sends 15-bit codes too)"""
    out = []
    for _, d, strategy, _, trees in H.designed():
        for level in (1, 6, 9):
            out.append((d, oracle.deflate(d, level=level, strategy=strategy)))
        for zs in (zlib.Z_HUFFMAN_ONLY, zlib.Z_DEFAULT_STRATEGY):
            out.append((d, _zlib_raw(d, zs)))
    return out


def _both(z, comp, caps):
    a = _run_plan(z, comp, caps)
    b = _serial(_run_plan, z, comp, caps)
    assert a[5]["parallel"] == 1 and b[5]["parallel"] == 0
    return a, b


def _long_codes(stream):
    blocks, _, _ = H.parse(stream)
    return sum(1 for b in blocks if b["type"] == 2 and (max(b["lit"]) == 15 or max(b["dist"]) == 15))


def test_emu_inflate_designed_streams(z, oracle):
    """both kernels on every stream: bytes, status, bytes used and restart points equal each other and the input"""
    items = _streams(oracle)
    assert sum(_long_codes(c) > 0 for _, c in items) >= 12
    comp, want = [c for _, c in items], [d for d, _ in items]
    a, b = _both(z, comp, [len(d) for d in want])
    assert a[0] == want and b[0] == want
    assert not a[1].any() and not b[1].any()
    assert [int(u) for u in a[2]] == [len(c) for c in comp] == [int(u) for u in b[2]]
    assert list(a[3]) == list(b[3]) and list(a[4]) == list(b[4])


def _multi_mib(oracle):
    """multi-MiB streams in which every third block has a 15-bit code: a 16 KiB literal chain under HUFFMAN_ONLY (one block
    that needs the repair), then 32 KiB of random bytes (two blocks), over and over.  The random blocks keep the stream
    within the pipeline's round pool: every block takes at least one batch of four rounds, and the pool gives a stream
    four rounds per 8 KiB of input, so a stream made of chain blocks alone (about 5 KiB each) would use it up and go to
    the serial kernel whole."""
    rng = datagen.Rng(0x15B)
    data = b"".join(H.literal_chain(16 + k % 3, seed=k, block=True) + rng.bytes(32768).tobytes() for k in range(40))
    return [(data, oracle.deflate(data, level=6, strategy=H.HUFFMAN_ONLY)), (data, _zlib_raw(data, zlib.Z_HUFFMAN_ONLY))]


def test_inflate_multi_mib_streams_run_in_parallel(z, oracle):
    """k_find / k_dec1 / k_dec2 with many segments per stream, a third of the blocks with 15-bit codes"""
    items = _multi_mib(oracle)
    comp, want = [c for _, c in items], [d for d, _ in items]
    assert all(len(d) > 1 << 20 for d in want) and _long_codes(comp[0]) == 40
    a, b = _both(z, comp, [len(d) for d in want])
    assert a[5]["handed_back"] == 0 and a[5]["segments"] > 3 * len(comp), a[5]
    assert a[0] == want and b[0] == want and not a[1].any() and not b[1].any()
    assert [int(u) for u in a[2]] == [len(c) for c in comp] == [int(u) for u in b[2]]
    assert list(a[3]) == list(b[3]) and list(a[4]) == list(b[4])


def _truncation_cases(oracle):
    """streams whose last bytes are 15-bit codes: the rarest literals of a repaired chain go last"""
    d = H.literal_chain(18, rare_last=True)
    c = oracle.deflate(d, level=6, strategy=H.HUFFMAN_ONLY)
    blocks, _, _ = H.parse(c)
    assert max(blocks[-1]["lit"]) == 15 and ("lit" in [t for _, t in H.limited_trees(blocks)])
    return d, c


def test_emu_truncated_inside_long_codes(z, oracle):
    """cut at every byte of the last 64: status, bytes and bytes used agree between both kernels and the oracle's
    Inflater -- a cut inside a 15-bit code is "needs input", not a data error"""
    d, c = _truncation_cases(oracle)
    cuts = [c[:len(c) - k] for k in range(1, 65)]
    a, b = _both(z, cuts, [len(d)] * len(cuts))
    for i, cut in enumerate(cuts):
        o = oracle.Inflater(nowrap=True)
        o.set_input(cut)
        got = bytearray()
        while True:
            r = o.inflate(1 << 16)
            if not r:
                break
            got += r
        got, rem = bytes(got), o.remaining_input
        assert o.needs_input and not o.finished
        assert int(a[1][i]) == int(b[1][i]) and int(a[1][i]) & 0xFF == 8, (i, int(a[1][i]), int(b[1][i]))
        assert a[0][i] == b[0][i] == got, i
        assert int(a[2][i]) == int(b[2][i]) == len(cut) - rem, (i, int(a[2][i]), int(b[2][i]), rem)


def test_inflater_fed_in_pieces(z, oracle):
    """the Inflater handle fed 1-7 bytes at a time gives what the oracle's Inflater gives for the same pieces"""
    d, c = _truncation_cases(oracle)
    dist = H.distance_chain(17)
    for data, comp in ((d, c), (dist, oracle.deflate(dist, level=6))):
        rnd = random.Random(len(comp))
        g, o = z.Inflater(True), oracle.Inflater(nowrap=True)
        got, ref, buf, pos = bytearray(), bytearray(), bytearray(1 << 15), 0
        while pos < len(comp):
            k = rnd.randint(1, 7)
            piece = comp[pos:pos + k]
            pos += k
            g.SetInput(piece)
            o.set_input(piece)
            while True:
                n = g.Inflate(buf)
                got += buf[:n]
                r = o.inflate(1 << 15)
                ref += r
                if n == 0 and not r:
                    break
            assert len(got) == len(ref) and g.IsNeedingInput == o.needs_input and g.IsFinished == o.finished, pos
        assert bytes(got) == bytes(ref) == data
        assert g.IsFinished and o.finished
        assert g.TotalIn == o.total_in == len(comp) and g.RemainingInput == o.remaining_input == 0
