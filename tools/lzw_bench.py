"""LZW (.Z) decompression on the GPU: GB/s of output and per-kernel times for two workloads.
- 1024 x 256 KiB datagen.silesia_mix streams (the batch shape).
- One 256 MiB datagen.log_stream (a single large stream).
Both are compressed with the compress(1)-format encoder of tests/cpu_model/lzw_model.cpp at 16 bits, block mode.

Each workload is timed two ways: device-resident (LzwPlan.run on device buffers, CUDA events) and end to end through
b200z_lzw_batch (host buffers in and out, host clock).  The single-thread decode time of the LzwInputStream restatement
(C++) is printed beside them as the proxy for the C# path.  The card name and power limit are printed in the same run.

    python tools/lzw_bench.py [--reps 5] [--small]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import lzw_ref as R  # noqa: E402
import sharpziplib_b200 as z  # noqa: E402
from sharpziplib_b200 import datagen  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def device_resident(streams, outs_len, reps):
    p = z.LzwPlan([len(s) for s in streams], outs_len)
    blob = np.zeros(p.in_bytes, np.uint8)
    for i, s in enumerate(streams):
        blob[p.in_offsets[i]:p.in_offsets[i] + len(s)] = np.frombuffer(s, np.uint8)
    n = len(streams)
    d_in = torch.from_numpy(blob).cuda()
    d_out = torch.empty(p.out_bytes, dtype=torch.uint8, device="cuda")
    ol = torch.zeros(n, dtype=torch.int64, device="cuda")
    st = torch.zeros(n, dtype=torch.int32, device="cuda")
    p.run(d_in, d_out, ol, st)  # warm-up
    torch.cuda.synchronize()
    assert not st.any() and ol.cpu().tolist() == list(outs_len)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        p.run(d_in, d_out, ol, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    p.set_timing(True)
    p.run(d_in, d_out, ol, st)  # a run of its own for the per-kernel times
    torch.cuda.synchronize()
    kt = p.timings()
    stats = p.stats()
    out = d_out.cpu().numpy()
    p.close()
    return ms, kt, stats, out


def end_to_end(streams, outs_len, reps):
    z.lzw_batch(streams, outs_len)  # warm-up: the pipeline of this shape is cached
    t = time.perf_counter()
    for _ in range(reps):
        outs, status, _ = z.lzw_batch(streams, outs_len)
    ms = (time.perf_counter() - t) * 1e3 / reps
    assert not status.any()
    return ms, outs


def run(name, data, reps):
    t = time.perf_counter()
    streams = [R.encode(d, 16) for d in data]
    enc_s = time.perf_counter() - t
    total = sum(len(d) for d in data)
    comp = sum(len(s) for s in streams)
    t = time.perf_counter()
    for s, d in zip(streams, data):
        r = R.decode(s)
        assert r.kind == 0 and len(r.out) == len(d)
    oracle_s = time.perf_counter() - t
    lens = [len(d) for d in data]
    ms, kt, stats, out = device_resident(streams, lens, reps)
    e2e_ms, outs = end_to_end(streams, lens, reps)
    assert outs == data, "end-to-end output differs from the input"
    scan_ms = kt.get("k_lzw_scan", float("nan"))
    res = {
        "workload": name, "streams": len(data), "output_bytes": total, "compressed_bytes": comp,
        "device_resident": {"ms": round(ms, 3), "gbs": round(total / ms / 1e6, 2)},
        "end_to_end_b200z_lzw_batch": {"ms": round(e2e_ms, 3), "gbs": round(total / e2e_ms / 1e6, 2)},
        "kernels_ms": {k: round(v, 3) for k, v in kt.items()},
        "scan_codes_per_s": round(stats["codes"] / (scan_ms / 1e3)) if scan_ms == scan_ms and scan_ms > 0 else None,
        "stats": stats,
        "cpu_proxy_single_thread": {"what": "C++ restatement of LzwInputStream (tests/cpu_model/lzw_model.cpp), one thread",
                                    "s": round(oracle_s, 3), "gbs": round(total / oracle_s / 1e9, 3)},
        "encode_s": round(enc_s, 2),
    }
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--small", action="store_true", help="64 x 64 KiB and one 8 MiB stream (a quick check)")
    a = ap.parse_args()
    z.init(0)
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name()}), flush=True)
    n, size, big = (64, 64 << 10, 8 << 20) if a.small else (1024, 256 << 10, 256 << 20)
    run("silesia_mix %d x %d KiB" % (n, size >> 10), [datagen.silesia_mix(i, size).tobytes() for i in range(n)], a.reps)
    run("log_stream %d MiB" % (big >> 20), [datagen.log_stream(big).tobytes()], a.reps)


if __name__ == "__main__":
    main()
