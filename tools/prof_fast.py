"""Small fixed workload for ncu captures of k_fast: NS x 256 KiB Silesia-mix at LEVEL (default 132 streams, one per H100 SM, level 1), two runs."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import sharpziplib_b200 as z  # noqa: E402
from sharpziplib_b200 import datagen  # noqa: E402

z.init(0)
ns, level = int(os.environ.get("NS", "132")), int(os.environ.get("LEVEL", "1"))
d_np = [datagen.silesia_mix(i % 32, 262144, config=5) for i in range(ns)]
plan = z.DeflatePlan([a.size for a in d_np], level=level)
h = np.zeros(plan.in_bytes, dtype=np.uint8)
for o, a in zip(plan.in_offsets, d_np):
    h[o:o + a.size] = a
d_in = torch.from_numpy(h).cuda()
d_out = torch.empty(plan.out_bytes, dtype=torch.uint8, device="cuda")
dl = torch.zeros(ns, dtype=torch.int64, device="cuda")
ds = torch.zeros(ns, dtype=torch.int32, device="cuda")
for _ in range(2):
    plan.run(d_in, d_out, dl, ds)
    torch.cuda.synchronize()
print("status", int(ds.abs().sum()), "clen", int(dl.sum()))
