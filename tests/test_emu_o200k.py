"""CPU: the o200k split (k_split_reduce<WITH_B, 3> with its last-block scan of the tile aggregates and
k_split_apply<TOKENS, WITH_B, 3>, in both TOKENS and both WITH_B forms, and every training and encode path that reaches them) on the SIMT emulator (tests/emu/, as
tests/test_emu_encode_docs.py does): the GPU tests of tests/test_gpu_zz_o200k.py run against the emulator build with a random
thread interleaving and the blocks of a grid on three OS threads."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
TEST = os.path.join("tests", "test_gpu_zz_o200k.py")


def test_emu_o200k_random_order_parallel_blocks():
    sys.path.insert(0, EMU)
    import build_emu
    env = dict(os.environ, BPE_LIB_PATH=build_emu.build(), BPE_TEST_SMALL="1", EMU_SMS="2", PYTHONDONTWRITEBYTECODE="1",
               EMU_ORDER="random", EMU_PAR="3")
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", TEST]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3600)
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-6000:]
