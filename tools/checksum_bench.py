"""The three checksum kinds on the GPU (0 = CRC-32, 1 = Adler-32, 2 = CRC-32/BZIP2), in the shape of the reference's own
checksum benchmarks (benchmark/.../Checksum/*.cs): 256 MiB of `new Random(1).NextBytes` (restated in the oracle), one Update
over all of it, and 256 Updates of 1 MiB with a running value.

Each kind and shape is timed three ways:
- host buffer, end to end: Crc32 / Adler32 / BZip2Crc.Update (copy to the device, reduce, copy the value back), host clock;
- device-resident: b200z_checksum_batch_device on a device blob, CUDA events (the 256 Updates are 256 calls, each starting
  from the value the one before left on the device; a batch of 256 independent 1 MiB streams in one call is reported too);
- the oracle on one host core: the C++ restatements of Crc32 and Adler32 (oracle/) and of BZip2Crc
  (tests/cpu_model/bzip2crc_model.cpp).
Every path's value is checked against the oracle's.  The card name and power limit are printed in the same run.

    python tools/checksum_bench.py [--reps 5] [--mib 256]
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

import bzip2crc_ref  # noqa: E402
import oracle_lib as O  # noqa: E402
import sharpziplib_b200 as z  # noqa: E402

MiB = 1 << 20
KINDS = {0: ("Crc32", z.Crc32), 1: ("Adler32", z.Adler32), 2: ("BZip2Crc", z.BZip2Crc)}
INIT = {0: 0, 1: 1, 2: 0}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def oracle_update(kind, value, a):
    if kind == 0:
        return O.crc32_update(value, a)
    if kind == 1:
        return O.adler32_update(value, a)
    return bzip2crc_ref.oracle(a, value)


def timed(fn, reps):
    """best and median of `reps` runs of fn(), in ms, and its last result"""
    fn()  # warm-up
    ts, r = [], None
    for _ in range(reps):
        t = time.perf_counter()
        r = fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts), float(np.median(ts)), r


def host(kind, data, pieces):
    c = KINDS[kind][1]()
    step = data.size // pieces
    for k in range(pieces):
        c.Update(data, k * step, step)
    return c.Value


def device_calls(kind, blob, offs, lens, calls, v):
    """`calls` calls of b200z_checksum_batch_device over (offs, lens) split into equal groups, in order on one stream"""
    s = torch.cuda.current_stream().cuda_stream
    per = len(lens) // calls
    for k in range(calls):
        o, L = offs[k * per:(k + 1) * per], lens[k * per:(k + 1) * per]
        rc = z.lib().b200z_checksum_batch_device(kind, blob.data_ptr(), o.ctypes.data, L.ctypes.data, per, v.data_ptr(), s)
        assert rc == 0, z.lib().b200z_last_error()


def device(kind, blob, offs, lens, calls, reps):
    """ms per run (CUDA events around `reps` runs, after a warm-up) and the values of the last run"""
    v = torch.empty(len(lens) // calls, dtype=torch.int32, device="cuda")
    seed = torch.full_like(v, INIT[kind])

    def once():
        v.copy_(seed)
        device_calls(kind, blob, offs, lens, calls, v)
    once()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        once()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, [int(x) for x in v.cpu().numpy().view(np.uint32)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mib", type=int, default=256, help="input size in MiB (the reference benchmark's: 256)")
    a = ap.parse_args()
    z.init(0)
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name()}), flush=True)
    n = a.mib * MiB
    data = O.dotnet_random_bytes(1, n)
    blob = torch.from_numpy(data).cuda()
    one = (np.zeros(1, np.int64), np.full(1, n, np.int64))
    split = (np.arange(a.mib, dtype=np.int64) * MiB, np.full(a.mib, MiB, np.int64))
    for kind, (name, _) in KINDS.items():
        t = time.perf_counter()
        want = oracle_update(kind, INIT[kind], data)
        oracle_one_s = time.perf_counter() - t
        t = time.perf_counter()
        v = INIT[kind]
        for k in range(a.mib):
            v = oracle_update(kind, v, data[k * MiB:(k + 1) * MiB])
        oracle_split_s = time.perf_counter() - t
        assert v == want, (name, "oracle pieces", hex(v), hex(want))
        res = {"kind": kind, "checksum": name, "bytes": n, "value": "0x%08X" % want,
               "oracle_one_core": {"one_update_gbs": round(n / oracle_one_s / 1e9, 3),
                                   "updates_of_1mib_gbs": round(n / oracle_split_s / 1e9, 3)}}
        for shape, pieces in (("one_update", 1), ("updates_of_1mib", a.mib)):
            best, med, got = timed(lambda: host(kind, data, pieces), a.reps)
            assert got == want, (name, shape, "host", hex(got), hex(want))
            res.setdefault("host_buffer_end_to_end", {})[shape] = {"ms_best": round(best, 3), "ms_median": round(med, 3),
                                                                    "gbs_best": round(n / best / 1e6, 2)}
        for shape, (offs, lens), calls in (("one_update", one, 1), ("updates_of_1mib", split, a.mib)):
            ms, got = device(kind, blob, offs, lens, calls, a.reps)
            assert got == [want], (name, shape, "device", got, hex(want))
            res.setdefault("device_resident", {})[shape] = {"ms": round(ms, 3), "gbs": round(n / ms / 1e6, 2)}
        ms, got = device(kind, blob, split[0], split[1], 1, a.reps)
        assert got == [oracle_update(kind, INIT[kind], data[k * MiB:(k + 1) * MiB]) for k in range(a.mib)], (name, "batch")
        res["device_resident"]["batch_of_1mib_streams"] = {"ms": round(ms, 3), "gbs": round(n / ms / 1e6, 2)}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
