"""CPU: the texts past a boundary B of tests/test_gpu_zz_beyond_32bit.py on the SIMT emulator (tests/emu/, as
tests/test_emu_train_specials.py does), at B = 2^22 (BPE_TEST_SMALL): the plain loop, train_from_file, train_from_iterator,
encode_file, decode and an encode without merges, against the oracle built from the blocks.  This checks the plumbing and
the oracle before an H100 runs them past 2^31 and 2^32; it cannot check 32-bit arithmetic itself.  The GPU tests run
against the emulator build with a random thread interleaving and the blocks of a grid on three OS threads."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
TEST = os.path.join("tests", "test_gpu_zz_beyond_32bit.py")


def test_emu_beyond_32bit_random_order_parallel_blocks():
    sys.path.insert(0, EMU)
    import build_emu
    env = dict(os.environ, BPE_LIB_PATH=build_emu.build(), BPE_TEST_SMALL="1", EMU_SMS="2", PYTHONDONTWRITEBYTECODE="1",
               EMU_ORDER="random", EMU_PAR="3")
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", TEST]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=2400)
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout and "skipped" not in p.stdout, p.stdout[-6000:]
