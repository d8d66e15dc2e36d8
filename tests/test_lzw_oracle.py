"""CPU tier: the LzwInputStream restatement and the compress(1)-format encoder of tests/cpu_model/lzw_model.cpp -- round
trips, an independent decoder (gzip -dc), independence from how the base stream's Read returns data, and every quirk of
the reference on a hand-built stream."""
import shutil
import subprocess

import numpy as np
import pytest

import lzw_ref as R
from lzw_quirks import QUIRKS, zeros_stream


def _data():
    rng = np.random.default_rng(3)
    text = b"".join(rng.choice([b"hour2890 ", b"09n ", b"GNSS ", b"observation\n", b"lzw "], 20000))
    return [text, bytes(70000), bytes(rng.integers(0, 256, 50000, dtype=np.uint8)), bytes(range(256)) * 300, b"x", b""]


CONFIGS = [(mb, True, 0) for mb in range(9, 17)] + [(mb, False, 0) for mb in (9, 12, 16)] + [(12, True, 1), (16, True, 255)]


@pytest.mark.parametrize("max_bits,block,every", CONFIGS)
def test_encoder_round_trips_through_the_model(max_bits, block, every):
    for d in _data():
        r = R.decode(R.encode(d, max_bits, block, every))
        assert r.kind == 0 and r.out == d


@pytest.mark.skipif(shutil.which("gzip") is None, reason="no gzip")
@pytest.mark.parametrize("max_bits,block,every", [(12, True, 0), (13, True, 0), (16, True, 0), (16, False, 0), (16, True, 100)])
def test_gzip_agrees(max_bits, block, every):
    for d in _data()[:4]:
        s = R.encode(d, max_bits, block, every)
        assert subprocess.run(["gzip", "-dc"], input=s, capture_output=True, check=True).stdout == d


@pytest.mark.parametrize("sizes", [[1], [7], [8191], "random"])
def test_base_stream_read_sizes_do_not_matter(sizes):
    rng = np.random.default_rng(11)
    if sizes == "random":
        sizes = [int(x) for x in rng.integers(1, 9000, 97)]
    streams = [R.encode(d, mb, True, ev) for d in _data()[:4] for mb, ev in ((9, 0), (12, 0), (16, 3), (16, 0))]
    streams += [s for _, s in QUIRKS if len(s) > 3]
    for s in streams:
        a, b = R.decode(s), R.decode(s, sizes)
        assert (a.kind, a.a, a.b, a.out, a.decoded) == (b.kind, b.a, b.b, b.out, b.decoded)


EXPECTED = {  # name: (kind, a, b, output)
    "empty": (1, 0, 0, b""),
    "one_byte": (1, 0x1F, 0, b""),
    "magic_only": (6, 1, 0, b""),
    "bad_magic": (1, 0x1F, 0x9E, b""),
    "max_bits_17": (2, 17, 0, b""),
    "reserved_bits": (3, 0, 0, b""),
    "max_bits_7": (6, 1, 0, b""),
    "max_bits_8_literals": (0, 0, 0, b"ABCD"),
    "max_bits_8_kwk": (0, 0, 0, b"AAAB"),
    "max_bits_8_kwk_on_kwk": (6, 4, 0, b"AAA"),
    "max_bits_8_nonblock_kwk_on_kwk": (6, 4, 0, b"AAA"),
    "max_bits_9_to_10": (5, 600, 512, None),
    "first_code_clear": (4, 256, 0, b""),
    "clear_every_code": (0, 0, 0, b"ABCDEEEF"),
    "clear_then_kwk_code": (0, 0, 0, b"ABCCC"),
    "kwk_every_width": (0, 0, 0, None),
    "kwk_nonblock_256": (0, 0, 0, b"AAAAAAB"),
    "code_gt_free_ent": (5, 300, 259, b"ABC"),
    "truncated_in_code": (0, 0, 0, b"ABABC"),
    "truncated_after_pad": (0, 0, 0, b"AB"),
    "truncated_before_pad": (6, 2, 0, b"AB"),
    "trailing_bits": (0, 0, 0, b"ABC"),
}


@pytest.mark.parametrize("name", [n for n, _ in QUIRKS])
def test_quirk(name):
    s = dict(QUIRKS)[name]
    kind, a, b, out = EXPECTED[name]
    r = R.decode(s, out_chunk=1)
    assert (r.kind, r.a, r.b) == (kind, a, b), r
    assert len(r.out) == r.decoded
    if out is not None:
        assert r.out == out
    if name == "max_bits_9_to_10":
        assert r.out[:301] == b"a" + b"b" * 300 and len(r.out) > 301
    if name == "kwk_every_width":
        assert len(r.out) > 65000


def test_error_surfaces_on_the_read_that_reaches_it():
    s = dict(QUIRKS)["code_gt_free_ent"]  # 3 bytes, then the bad code
    assert R.decode(s, out_chunk=3).out == b"ABC"   # Read(3) returns them; the next Read throws
    r = R.decode(s, out_chunk=4)
    assert r.kind == 5 and r.out == b"" and r.decoded == 3  # Read(4) reaches the code and throws


def test_zeros_stream_builder():
    for n in (2, 3, 1000, 65280 * 65281 // 2 + 70000):
        r = R.decode(zeros_stream(n))
        assert r.kind == 0 and len(r.out) == n and not any(r.out)
