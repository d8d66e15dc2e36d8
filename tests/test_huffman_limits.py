"""CPU tier: DEFLATE's Huffman length limits (15 bits, 7 for the code-length code).  Inputs built so that an optimal tree
would be deeper than the limit make the encoder run the length-limit repair of `build_tree` (b200z_core.cuh); a plain
Python parser (tests/huffman_limits.py) proves that each of them reaches it, and the CPU model of the kernels and the
kernels themselves on the CUDA emulator must give the oracle's bytes for them."""
import os
import subprocess
import sys

import pytest

import huffman_limits as H
from test_cpu_model import model  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DESIGNED = H.designed()


@pytest.mark.parametrize("case", DESIGNED, ids=[c[0] for c in DESIGNED])
def test_designed_inputs_reach_the_length_limit(oracle, case):
    """(a) lengths within the limits and Kraft sums of at most 1, (b) the repair really ran: the emitted code costs more
    than an optimal one for the same counts, (c) a code exactly at the limit, (d) the stream decodes to the input"""
    name, d, strategy, levels, trees = case
    for level in levels:
        blocks = H.check_stream(oracle.deflate(d, level=level, strategy=strategy), d, [(0, t) for t in trees])
        assert len(blocks) == 1 and blocks[0]["type"] == 2, (name, level)
        if not trees:   # 15 deep and optimal: the limit is reached without a repair
            assert H.limited_trees(blocks) == [] and max(blocks[0]["lit"]) == 15, level
        for t in trees:  # the repaired codes are complete (the block finder of the parallel inflate takes only those)
            assert H.kraft(blocks[0][t]) == 1 << 15, (name, level, t)


def test_the_designs_are_exact(oracle):
    """the generators give exactly the designed counts: what the parser counts in the oracle's block"""
    for n in (15, 16, 17, 18):
        blocks, _, _ = H.parse(oracle.deflate(H.literal_chain(n), level=6, strategy=H.HUFFMAN_ONLY))
        counts = sorted(c for c in blocks[0]["lit_counts"] if c)
        assert counts == sorted(H.fib_counts(n) + [1]), n
    blocks, _, _ = H.parse(oracle.deflate(H.distance_chain(17), level=6))
    assert blocks[0]["dist_counts"][:17] == [1] + H.fib_counts(16)
    assert not any(blocks[0]["dist_counts"][17:])


@pytest.mark.parametrize("case", DESIGNED, ids=[c[0] for c in DESIGNED])
def test_cpu_model_matches_the_oracle(model, oracle, case):  # noqa: F811
    """build_tree as the kernels run it (the CPU model of b200z_core.cuh) on every designed input: levels 1-9, all three
    strategies, Finish() alone and Flush() then Finish()"""
    name, d, _, _, _ = case
    for level in range(1, 10):
        for strategy in (0, 1, 2):
            assert model(d, level, strategy) == oracle.deflate(d, level=level, strategy=strategy), (name, level, strategy)
            assert model(d, level, strategy, 1) == oracle.deflate(d, level=level, strategy=strategy, pattern=1), \
                (name, level, strategy)


def placements():
    """the 18-deep literal chain as the first block, after 32 KiB of text (two whole blocks under HUFFMAN_ONLY) with text
    behind it, and as the last block of the stream"""
    chain, t = H.literal_chain(18, seed=1, block=True), H.text(60000)
    return [("first", chain + t[:40000], 0), ("middle", t[:32768] + chain + t[32768:], 2),
            ("last", t[:32768] + H.literal_chain(18, seed=1), 2)]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_chain_among_other_blocks(model, oracle, where):  # noqa: F811
    _, d, block = next(p for p in placements() if p[0] == where)
    for level in (1, 4, 6, 9):
        ref = oracle.deflate(d, level=level, strategy=H.HUFFMAN_ONLY)
        H.check_stream(ref, d, [(block, "lit")])
        assert model(d, level, H.HUFFMAN_ONLY) == ref, level
        assert model(d, level, H.HUFFMAN_ONLY, 1) == oracle.deflate(d, level=level, strategy=H.HUFFMAN_ONLY, pattern=1), level


def test_kernels_on_the_emulator():
    """the GPU tier's small cases on the CUDA emulator: k_plan builds these trees, both inflate kernels decode them"""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"),
                        os.path.join(ROOT, "tests", "test_gpu_huffman_limits.py"), "-k", "emu"],
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and " passed" in r.stdout and "deselected" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
