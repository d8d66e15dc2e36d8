"""CPU tier: the small cases of test_gpu_lzw.py (LZW kernels against the LzwInputStream restatement) on the CUDA emulator, in
the default and in a reversed thread order.  In a subprocess: the emulator library never shares a process with tests of the
real one."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_lzw_cases_on_the_emulator(order):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"), "-k",
                        "quirk or clear_every or nomem or plan_run or pack", os.path.join(ROOT, "tests", "test_gpu_lzw.py")],
                       capture_output=True, text=True, timeout=3000, env=dict(os.environ, B200Z_EMU_ORDER=order))
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
