"""One long GZipOutputStream on the GPU: a seeded C4-style log stream of --gib GiB in 1 MiB writes.  Prints one JSON line:
throughput over the whole stream (host side included), the time to the first compressed byte behind the gzip header, the
device memory in use between writes (torch.cuda.mem_get_info after every write: a plan's workspace lives only inside the
Deflate() call that runs it, so this is what stays allocated), the compressed size, and the card's name and power limit.

    python tools/stream_deflate_bench.py --gib 3 [--level 6]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=3.0)
    ap.add_argument("--level", type=int, default=6)
    a = ap.parse_args()
    import torch
    import sharpziplib_b200 as z
    from sharpziplib_b200 import datagen
    z.init(0)
    total = int(a.gib * (1 << 30))
    pool = datagen.log_stream(96 << 20).tobytes()  # cycled with moving offsets: generating GiBs of lines takes minutes
    free0, dev_total = torch.cuda.mem_get_info()
    state = {"first": None, "out": 0, "peak": 0}

    class Sink:
        def write(self, b):
            state["out"] += len(b)
            if state["first"] is None and state["out"] > 10:  # GetHeader writes 10 bytes at the first Write
                state["first"] = time.perf_counter()

    def sample():
        free, _ = torch.cuda.mem_get_info()
        state["peak"] = max(state["peak"], free0 - free)

    g = z.GZipOutputStream(Sink(), level=a.level)
    g.ModifiedTime = 0
    t0 = time.perf_counter()
    pos, k = 0, 0
    while pos < total:
        off = (k * 7919 * 4096) % (len(pool) - (1 << 20))
        m = min(1 << 20, total - pos)
        g.Write(pool[off:off + m])
        sample()
        pos += m
        k += 1
    g.Finish()
    sample()
    secs = time.perf_counter() - t0
    name, power = card()
    print(json.dumps({"bytes_in": total, "bytes_out": state["out"], "level": a.level, "seconds": round(secs, 3),
                      "gb_per_s": round(total / secs / 1e9, 4), "first_output_s": round(state["first"] - t0, 3),
                      "device_mem_between_writes_gib": round(state["peak"] / 2 ** 30, 3), "device_mem_gib": round(dev_total / 2 ** 30, 1),
                      "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
