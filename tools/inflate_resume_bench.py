"""InflaterInputStream throughput with 4 KiB and 1 MiB buffers on two 64 MiB streams: the level-6 oracle stream bench.py
reads back (bench.py's deflate-leg buffers, blocks of 16384 symbols) and one static block of 64 MiB built by
tests/test_gpu_inflate_resume.py.  With --parent-lib PATH the same reads run on another build of libb200z.so (the commit
in front of a change), alternating with this tree's library in the same process; a read that would take longer than
--budget seconds stops there and reports the rate of what it read.  Prints the card's name and power limit and one JSON
line.

    python tools/inflate_resume_bench.py [--parent-lib sharpziplib_b200/csrc/_build/parent/libb200z.so] [--reps 2]"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def load(path):
    from sharpziplib_b200 import _lib
    L = C.CDLL(path)
    for name, (res, args) in _lib._SIGS.items():
        f = getattr(L, name, None)
        if f is not None:
            f.restype = res
            f.argtypes = args
    return L


def read_rate(z, comp, orig, buffer_size, budget):
    r = z.InflaterInputStream(io.BytesIO(comp), z.Inflater(True), bufferSize=buffer_size)
    back = bytearray()
    t = time.perf_counter()
    while len(back) < len(orig) and time.perf_counter() - t < budget:
        chunk = r.read(1 << 16)
        if not chunk:
            break
        back += chunk
    dt = time.perf_counter() - t
    assert bytes(back) == orig[:len(back)], "InflaterInputStream bytes differ"
    return {"gbs": round(len(back) / dt / 1e9, 4), "bytes": len(back), "seconds": round(dt, 3), "complete": len(back) == len(orig)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--budget", type=float, default=60.0)
    args = ap.parse_args()
    import oracle_lib as O
    import sharpziplib_b200 as z
    from sharpziplib_b200 import _lib, datagen
    import test_gpu_inflate_resume as T
    print("card:", card(), flush=True)
    blob = b"".join(datagen.silesia_mix(i, 262144, config=3).tobytes() for i in range(256))
    O.build()
    streams = {"oracle_l6_64MiB": (O.deflate(blob, level=6), blob), "one_static_block_64MiB": T.build_static(O, 64 << 20, seed=11)}
    libs = {"this": _lib.lib()}
    if args.parent_lib:
        libs["parent"] = load(args.parent_lib)
    z.init(0)
    res = {}
    for rep in range(args.reps):
        for name, (comp, orig) in streams.items():
            for bs in (4096, 1 << 20):
                for which, L in libs.items():
                    _lib._lib = L
                    if which == "parent":
                        L.b200z_init(0)
                    r = read_rate(z, comp, orig, bs, args.budget)
                    res.setdefault("%s/%s/%s" % (name, "4KiB" if bs == 4096 else "1MiB", which), []).append(r)
                    print(rep, name, bs, which, r, flush=True)
    _lib._lib = libs["this"]
    print(json.dumps({"card": card(), "results": res}))


if __name__ == "__main__":
    main()
