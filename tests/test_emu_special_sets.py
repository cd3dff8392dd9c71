"""CPU: special-token sets of up to 65,536 specials (the trie matcher k_special_find, the 16-bit candidate index, the
seeding of large sets into the encode memo, the host trie of the re-pick and the piece cuts) on the SIMT emulator
(tests/emu/, as tests/test_emu_train_specials.py does): the GPU tests of tests/test_gpu_zz_special_sets.py run against the
emulator build with a random thread interleaving and the blocks of a grid on three OS threads, and once more against the
UBSan build (alignment, shift counts, array bounds)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
TEST = os.path.join("tests", "test_gpu_zz_special_sets.py")


def _run(lib, extra_env, timeout=2400):
    env = dict(os.environ, BPE_LIB_PATH=lib, BPE_TEST_SMALL="1", EMU_SMS="2", PYTHONDONTWRITEBYTECODE="1", **extra_env)
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", TEST]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-6000:]


def test_emu_special_sets_random_order_parallel_blocks():
    sys.path.insert(0, EMU)
    import build_emu
    _run(build_emu.build(), {"EMU_ORDER": "random", "EMU_PAR": "3"})


def test_emu_special_sets_sanitized():
    out = subprocess.run([sys.executable, os.path.join(EMU, "build_emu.py"), "--force"], cwd=ROOT, check=True, text=True,
                         stdout=subprocess.PIPE, env=dict(os.environ, EMU_SANITIZE="1")).stdout
    lib = out.strip().splitlines()[-1]
    assert lib.endswith("_ubsan.so")
    ubsan = subprocess.run(["g++", "-print-file-name=libubsan.so"], check=True, text=True, stdout=subprocess.PIPE).stdout.strip()
    _run(lib, {"LD_PRELOAD": ubsan})
