"""Many compressed streams that arrive in pieces: an InflaterSet (one write() per round, every stream's next piece in it)
against the same number of Inflater handles driven round robin with the same pieces, alternating in one process.
Workloads: 256 streams of 16 MiB and 1024 streams of 1 MiB, level-6 oracle streams of silesia_mix data (a few distinct
streams, repeated), each fed in 4 KiB, 64 KiB and 1 MiB pieces.  A way that would take longer than --budget seconds stops
after the round it is in and reports the rate of what it decoded; the outputs of both ways are compared over what both
decoded.  Prints the card's name and power limit, then one JSON line: per workload and piece size GB/s of output for each
way, host-to-device bytes per output byte of the set, plans created and plans run.

    python tools/inflate_streams_bench.py [--budget 20] [--workloads 256x16,1024x1] [--pieces 4096,65536,1048576]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # (reported, not guessed)
        return "unknown (%s)" % e, "unknown"


def run_set(z, comp, piece, budget):
    from sharpziplib_b200 import _lib
    n = len(comp)
    s = z.InflaterSet(n, _lib.WRAP_RAW)
    got = [bytearray() for _ in range(n)]
    rounds = max(len(c) for c in comp) // piece + 1
    t = time.perf_counter()
    for r in range(rounds):
        s.write([c[r * piece:(r + 1) * piece] for c in comp])
        for i, b in enumerate(s.read()):
            got[i] += b
        if time.perf_counter() - t > budget:
            break
    dt = time.perf_counter() - t
    st = s.stats()
    s.close()
    out = sum(len(g) for g in got)
    return got, {"gbs": round(out / dt / 1e9, 4), "out_bytes": out, "seconds": round(dt, 3),
                 "h2d_per_out_byte": round(st["uploaded"] / max(out, 1), 4), "plans_created": st["created"],
                 "plans_run": st["plans"], "stream_runs": st["runs"], "complete": r == rounds - 1}


def run_handles(z, comp, piece, budget):
    n = len(comp)
    hs = [z.Inflater(True) for _ in range(n)]
    got = [bytearray() for _ in range(n)]
    buf = bytearray(4 << 20)
    rounds = max(len(c) for c in comp) // piece + 1
    t = time.perf_counter()
    for r in range(rounds):
        for i, c in enumerate(comp):
            p = c[r * piece:(r + 1) * piece]
            if not p or hs[i].IsFinished:
                continue
            hs[i].SetInput(p)
            while True:
                k = hs[i].Inflate(buf)
                if k == 0:
                    break
                got[i] += buf[:k]
        if time.perf_counter() - t > budget:
            break
    dt = time.perf_counter() - t
    out = sum(len(g) for g in got)
    return got, {"gbs": round(out / dt / 1e9, 4), "out_bytes": out, "seconds": round(dt, 3), "complete": r == rounds - 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget", type=float, default=20.0)
    ap.add_argument("--workloads", default="256x16,1024x1")
    ap.add_argument("--pieces", default="4096,65536,1048576")
    ap.add_argument("--distinct", type=int, default=4)
    args = ap.parse_args()
    import oracle_lib as O
    import sharpziplib_b200 as z
    from sharpziplib_b200 import datagen
    name, power = card()
    print("card: %s, power limit %s" % (name, power), flush=True)
    O.build()
    z.init(0)
    result = {"card": name, "power_limit": power, "runs": []}
    for wl in args.workloads.split(","):
        n, mib = (int(x) for x in wl.split("x"))
        uniq = [O.deflate(datagen.silesia_mix(i, mib << 20, config=3).tobytes(), level=6, nowrap=True) for i in range(args.distinct)]
        comp = [uniq[i % len(uniq)] for i in range(n)]
        for piece in (int(p) for p in args.pieces.split(",")):
            got_s, rs = run_set(z, comp, piece, args.budget)
            got_h, rh = run_handles(z, comp, piece, args.budget)
            for a, b in zip(got_s, got_h):
                k = min(len(a), len(b))
                assert bytes(a[:k]) == bytes(b[:k]), "set and handles decode different bytes"
            row = {"streams": n, "mib": mib, "piece": piece, "set": rs, "handles": rh}
            print(json.dumps(row), flush=True)
            result["runs"].append(row)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
