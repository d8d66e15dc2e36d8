"""CPU tier: the small Deflater set cases of test_gpu_deflate_streams.py (levels 0, 1 and 6, three streams, two of them
through two open runs, and a stream starting in the same plan as continuing ones at levels 0, 2, 3, 4 and 6) on the CUDA
emulator.  The emulator library is built with open runs of 100000 bytes instead of 4.25 MiB and plans of at most 250000
input bytes instead of 1 GiB, so that the same scripts run on small data and the set splits its due streams into several
plans; in a subprocess: the emulator library never shares a process with tests of the real one."""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUN_BYTES = 100000
PLAN_BYTES = 250000


def test_small_deflater_set_cases_on_the_emulator():
    with tempfile.TemporaryDirectory() as out:
        flags = "-DB200Z_SET_RUN_BYTES=%d -DB200Z_SET_PLAN_BYTES=%d" % (RUN_BYTES, PLAN_BYTES)
        env = dict(os.environ, B200Z_EMU_CXXFLAGS=flags, B200Z_EMU_OUT=out, B200Z_SET_RUN_BYTES=str(RUN_BYTES))
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cuda_emu", "run_emulated.py"), "-k", "small",
                            os.path.join(ROOT, "tests", "test_gpu_deflate_streams.py")], capture_output=True, text=True,
                           timeout=3000, env=env)
    assert r.returncode == 0 and "8 passed" in r.stdout and "failed" not in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
