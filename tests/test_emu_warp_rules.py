"""CPU: the warp collectives of the SIMT emulator (tests/emu/cuda_emu.h) and the warp folds of the kernels on it.

tests/emu/warp_rules.cpp is compiled against the emulator alone and runs one case per process.  Positive cases compare
__match_any_sync and full-mask shuffles after divergent work with a brute-force model, under every thread order the
emulator has.  Negative cases break one rule each — two call sites, two kinds, two masks meeting in one collective, a
lane outside its own mask, __activemask(), a full-mask match in a loop whose trip count differs per lane — and must stop
with that rule's report; a shuffle from an exited lane must read the guard fill.

tests/test_gpu_zz_warp_fold.py (every __match_any_sync fold of the kernels, on layouts where a warp's lanes leave a
segment at different trips) then runs against the emulator build with a random thread interleaving and the blocks of a
grid on three OS threads, and once more against the UBSan build."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
ORDERS = ["index", "reverse", "random"]


@pytest.fixture(scope="module")
def driver():
    out = os.path.join(EMU, "_build", "warp_rules")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    srcs = [os.path.join(EMU, f) for f in ("warp_rules.cpp", "cuda_emu.cpp", "cuda_emu.h")]
    if not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-I", EMU, srcs[0], srcs[1], "-o", out, "-lpthread"])
    return out


def _case(driver, name, order):
    env = dict(os.environ, EMU_ORDER=order)
    return subprocess.run([driver, name], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=300)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("name", ["match_full", "match_partial", "match_exited", "match_64bit", "reconverge"])
def test_collectives_match_the_model(driver, name, order):
    p = _case(driver, name, order)
    assert p.returncode == 0 and p.stdout.strip() == f"ok {name}", p.stderr[-3000:]


# each broken rule: the report's first line, and what it must name
BROKEN = {
    "two_sites": ("two call sites meet", ["kernel k_two_sites", "__syncwarp(mask 0xffffffff)", "warp_rules.cpp:"]),
    "two_kinds": ("two kinds of collective meet", ["kernel k_two_kinds", "__syncwarp", "__ballot_sync"]),
    "two_masks": ("two masks meet", ["kernel k_two_masks", "mask 0xffffffff", "mask 0xffff0000"]),
    "outside_mask": ("the calling lane is not in its own mask", ["kernel k_outside_mask", "lane 0 is at __syncwarp(mask 0xfffffffe)"]),
    "activemask": ("__activemask() called at", ["in kernel k_activemask"]),
    "loop_match": ("is deadlocked", ["kernel k_loop_match", "waits in __match_any_sync(mask 0xffffffff)"]),
}


@pytest.mark.parametrize("name", sorted(BROKEN))
def test_broken_rule_stops_the_kernel(driver, name):
    what, also = BROKEN[name]
    p = _case(driver, name, "random")
    assert p.returncode != 0 and "ok" not in p.stdout, p.stdout
    report = [ln for ln in p.stderr.splitlines() if ln.startswith("emu:")]
    assert report and what in report[0], p.stderr[-3000:]
    for s in also:
        assert s in p.stderr, (s, p.stderr[-3000:])
    others = {w for w, _ in BROKEN.values()} - {what}
    assert not any(o in p.stderr for o in others), p.stderr[-3000:]


def test_shuffle_from_an_exited_lane_reads_the_guard_fill(driver):
    for order in ORDERS:
        p = _case(driver, "shfl_exited", order)
        assert p.returncode == 0, p.stderr[-3000:]
        reads = [ln.split()[-1] for ln in p.stdout.splitlines() if " read " in ln]
        assert len(reads) == 32 and set(reads) == {"0xcdcdcdcd"}, p.stdout


def _run_fold_tests(lib, extra_env, timeout=1800):
    env = dict(os.environ, BPE_LIB_PATH=lib, BPE_TEST_SMALL="1", EMU_SMS="2", PYTHONDONTWRITEBYTECODE="1", **extra_env)
    env.pop("PYTEST_CURRENT_TEST", None)
    cmd = [sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu", "-p", "no:cacheprovider", os.path.join("tests", "test_gpu_zz_warp_fold.py")]
    p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-6000:]


def test_emu_warp_folds_random_order_parallel_blocks():
    sys.path.insert(0, EMU)
    import build_emu
    _run_fold_tests(build_emu.build(), {"EMU_ORDER": "random", "EMU_PAR": "3"})


def test_emu_warp_folds_sanitized():
    out = subprocess.run([sys.executable, os.path.join(EMU, "build_emu.py"), "--force"], cwd=ROOT, check=True, text=True,
                         stdout=subprocess.PIPE, env=dict(os.environ, EMU_SANITIZE="1")).stdout
    lib = out.strip().splitlines()[-1]
    assert lib.endswith("_ubsan.so")
    ubsan = subprocess.run(["g++", "-print-file-name=libubsan.so"], check=True, text=True, stdout=subprocess.PIPE).stdout.strip()
    _run_fold_tests(lib, {"LD_PRELOAD": ubsan})
