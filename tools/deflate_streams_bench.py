"""Many long streams that arrive in pieces: --streams streams of --mib MiB each, written in 1 MiB pieces round robin, every
stream finishing with its last piece.  Two ways, alternating in one process: a DeflaterSet (one write() per round, every
stream's piece in it) and --streams Deflater handles driven round robin as DeflaterOutputStream drives one.  The outputs
of the two are compared.  Prints a progress line behind each way, then one JSON line per corpus and level: GB/s of input for each way and each repetition, the
set's stats, and the card's name and power limit read in the same run.

    python tools/deflate_streams_bench.py [--streams 256] [--mib 64] [--levels 6,1] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # (reported, not guessed)
        return "unknown (%s)" % e, "unknown"


def streams_of(kind, n, size):
    """n streams of `size` bytes cut from one seeded pool at moving offsets (generating GiBs takes minutes)"""
    from sharpziplib_b200 import datagen
    pool_len = 96 << 20
    pool = (datagen.log_stream(pool_len) if kind == "log_stream" else datagen.silesia_mix(0, pool_len, config=3)).tobytes()
    assert size <= pool_len
    ring = memoryview(pool + pool)
    return [ring[(i * 7919 * 4096) % pool_len:][:size] for i in range(n)]


def run_set(z, streams, level, piece):
    n, size = len(streams), len(streams[0])
    outs = [[] for _ in range(n)]
    s = z.DeflaterSet(n, level=level)
    t0 = time.perf_counter()
    for pos in range(0, size, piece):
        last = pos + piece >= size
        s.write([st[pos:pos + piece] for st in streams], [2 if last else 0] * n)
        for i, b in enumerate(s.read()):
            outs[i].append(b)
    dt = time.perf_counter() - t0
    stats = s.stats()
    s.close()
    return dt, [b"".join(o) for o in outs], stats


def run_handles(z, streams, level, piece):
    n, size = len(streams), len(streams[0])
    outs = [[] for _ in range(n)]
    hs = [z.Deflater(level) for _ in range(n)]
    buf = bytearray(8 << 20)

    def drain(d, o):
        while True:
            k = d.Deflate(buf)
            if k <= 0:
                break
            o.append(bytes(buf[:k]))
    t0 = time.perf_counter()
    for pos in range(0, size, piece):
        for i in range(n):
            d = hs[i]
            d.SetInput(streams[i][pos:pos + piece])
            while not d.IsNeedingInput:
                drain(d, outs[i])
            if pos + piece >= size:
                d.Finish()
                drain(d, outs[i])
                hs[i] = d = None  # (a handle keeps pinned staging of its stream's size until it is destroyed)
    dt = time.perf_counter() - t0
    return dt, [b"".join(o) for o in outs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=256)
    ap.add_argument("--mib", type=float, default=64)
    ap.add_argument("--levels", default="6,1")
    ap.add_argument("--corpora", default="log_stream,silesia_mix")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import sharpziplib_b200 as z
    z.init(0)
    name, power = card()
    piece, size = 1 << 20, int(a.mib * (1 << 20))
    for kind in a.corpora.split(","):
        streams = streams_of(kind, a.streams, size)
        total = a.streams * size
        for level in [int(x) for x in a.levels.split(",")]:
            rec = {"corpus": kind, "level": level, "streams": a.streams, "mib_per_stream": a.mib, "piece": piece, "gpu": name,
                   "power_limit": power, "set_gbps": [], "handles_gbps": []}
            for _ in range(a.reps):
                dt, set_out, stats = run_set(z, streams, level, piece)
                rec["set_gbps"].append(round(total / dt / 1e9, 3))
                print(json.dumps({"corpus": kind, "level": level, "set_gbps": rec["set_gbps"][-1]}), flush=True)
                dt, h_out = run_handles(z, streams, level, piece)
                rec["handles_gbps"].append(round(total / dt / 1e9, 3))
                print(json.dumps({"corpus": kind, "level": level, "handles_gbps": rec["handles_gbps"][-1]}), flush=True)
                rec["equal"] = set_out == h_out
                rec["ratio"] = round(sum(len(o) for o in set_out) / total, 4)
                rec["stats"] = stats
                del set_out, h_out
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
