"""CPU: tests/emu/kernel_coverage.json (written by tests/emu/kernel_coverage.py; tests/conftest.py orders the GPU tests by it)
must know every kernel of minbpe_b200/csrc.  A kernel added without regenerating the map would leave the tests that
launch it classified from a stale map."""
import glob
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# kernels the emulator trace cannot reach: the step kernels of the sharded loop (tests/test_gpu_sharded.py needs torch CUDA
# tensors; tests/conftest.py classifies its tests by hand) and the NVLink exchange kernels
UNTRACED = {"k_commit_candidate", "k_pack_candidate", "k_present_init", "k_present_update", "k_tie_present",
            "k_xchg_apply", "k_xchg_cand", "k_xchg_probe"}


def _kernels():
    names = set()
    for f in glob.glob(os.path.join(ROOT, "minbpe_b200", "csrc", "*.cu*")) + glob.glob(os.path.join(ROOT, "minbpe_b200", "csrc", "*.inl")):
        src = open(f, encoding="utf-8").read()
        names |= set(re.findall(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\([^)]*\)\s+)?(?:void\s+)?(\w+)\s*\(", src))
    return names


def _map():
    with open(os.path.join(ROOT, "tests", "emu", "kernel_coverage.json")) as f:
        return json.load(f)


def test_every_kernel_is_in_the_coverage_map():
    names = _kernels()
    seen = {re.sub(r"<.*", "", k) for v in _map()["tests"].values() for k in v}
    assert UNTRACED <= names, sorted(UNTRACED - names)
    assert not (names - seen - UNTRACED), f"regenerate tests/emu/kernel_coverage.json: {sorted(names - seen - UNTRACED)}"
    assert not (seen - names), sorted(seen - names)


def test_hw_validated_set_matches_the_generator():
    import importlib.util
    spec = importlib.util.spec_from_file_location("kernel_coverage", os.path.join(ROOT, "tests", "emu", "kernel_coverage.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    hw = _map()["hw_validated"]
    assert hw == sorted(mod.HW_VALIDATED)
    assert {re.sub(r"<.*", "", k) for k in hw} <= _kernels()
