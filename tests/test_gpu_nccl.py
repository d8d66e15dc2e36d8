"""GPU tier: the static-table broadcast through NCCL inside the library (b200z_static_tables_broadcast), one process per
GPU under torchrun, on up to four GPUs.  NCCL takes one rank per device, so a one-GPU box runs a one-rank communicator:
the library's NCCL resolution, ncclBroadcast, copy back and table import all run, only the transfer between GPUs does not."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_static_tables_broadcast_through_the_librarys_nccl_call(z):
    import torch
    n = min(torch.cuda.device_count(), 4)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(n), "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tools", "nccl_broadcast_check.py")], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and r.stdout.count("ncclBroadcast ok") == n, (r.stdout[-2000:], r.stderr[-3000:])


def test_broadcast_rejects_a_missing_communicator(z):
    assert z.lib().b200z_static_tables_broadcast(None, 0, 0, None) == 1  # B200Z_E_ARG
