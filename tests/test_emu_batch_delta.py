"""CPU: tests/test_gpu_zz_batch_delta.py (k_merge_seg's statistics delta with direct shared counters and with the hashed
cache) on the SIMT emulator (tests/emu/), with a random thread interleaving and the blocks of a grid on three OS threads."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")


def test_emu_batch_delta_random_order_parallel_blocks():
    sys.path.insert(0, EMU)
    import build_emu
    env = dict(os.environ, BPE_LIB_PATH=build_emu.build(), BPE_TEST_SMALL="1", EMU_SMS="2", EMU_ORDER="random", EMU_PAR="3",
               PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider",
           os.path.join("tests", "test_gpu_zz_batch_delta.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-6000:]
