"""CPU tier: the small Inflater set cases of test_gpu_inflate_streams.py (every wrap and piece size, trailing bytes, a zlib
trailer fed byte by byte, preset dictionaries, corrupt and truncated streams next to good ones, output larger than a
plan's capacity, and plans split and reused) on the CUDA emulator.  The emulator library is built with plans of at most
200000 compressed and 4 MiB output bytes instead of 256 MiB and 4 GiB, so that the small cases split their due streams
into several plans; in a subprocess: the emulator library never shares a process with tests of the real one."""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_small_inflater_set_cases_on_the_emulator():
    with tempfile.TemporaryDirectory() as out:
        flags = "-DB200Z_INFLATE_SET_PLAN_BYTES=200000 -DB200Z_INFLATE_SET_PLAN_OUT=4194304"
        env = dict(os.environ, B200Z_EMU_CXXFLAGS=flags, B200Z_EMU_OUT=out)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"), "-k", "small",
                            os.path.join(ROOT, "tests", "test_gpu_inflate_streams.py")], capture_output=True, text=True,
                           timeout=3000, env=env)
    assert r.returncode == 0 and "8 passed" in r.stdout and "failed" not in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
