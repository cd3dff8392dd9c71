import json
import os
import sys

import pytest

# The GPU tests run the byte-pair histogram of iteration 0 with k_hist_dense, the library's default; tests/test_gpu_zz_hist.py
# — last group — selects the packed kernel and the automatic choice explicitly.
os.environ.setdefault("BPE_HIST_KERNEL", "2")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with -m gpu")


def pytest_sessionstart(session):
    """A checkout that has never been built (the libraries are git-ignored): build them once, as __graft_entry__.build() does.
    nvcc cross-compiles without a GPU; on a box without nvcc the tests that need the library fail with its loader's message."""
    so = os.path.join(ROOT, "minbpe_b200", "csrc", "libb200bpe.so")
    if os.path.exists(so):
        return
    import shutil
    if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
        import __graft_entry__
        __graft_entry__.build()


# GPU tests that cannot be traced on the emulator (they need torch CUDA tensors): classified by hand.  1 = reaches a kernel
# outside the hardware-validated set (k_xchg_*), 0 = kernels inside it.
_MANUAL_GPU_ORDER = {"test_step_api_world1[p2p]": 1, "test_step_api_world1[collective]": 0,
                     "test_step_api_world2_nccl[p2p]": 1, "test_step_api_world2_nccl[collective]": 0,
                     # left out of the coverage run for their size; both launch the split / training kernels only
                     "test_large_properties": 0, "test_piecewise_split_equals_whole": 0}


def pytest_collection_modifyitems(config, items):
    """For `pytest -x -m gpu`: order the GPU tests so that tests launching only kernels of the hardware-validated set come
    first and tests reaching any other kernel come last (map and set: tests/emu/kernel_coverage.json, written by
    tests/emu/kernel_coverage.py).  A kernel that misbehaves on real hardware then costs the tests behind it, not
    the ones that would have passed.  Order inside each group is unchanged; CPU tests are not touched."""
    path = os.path.join(ROOT, "tests", "emu", "kernel_coverage.json")
    if not os.path.exists(path):
        return
    with open(path) as f:
        cov = json.load(f)
    hw = set(cov["hw_validated"]) | set(cov.get("order_ignore", []))

    def group(item):
        if item.get_closest_marker("gpu") is None:
            return 0
        if item.name in _MANUAL_GPU_ORDER:
            return _MANUAL_GPU_ORDER[item.name]
        kernels = cov["tests"].get(item.nodeid)
        if kernels is None:
            kernels = cov["tests"].get("tests/" + item.nodeid)
        if kernels is None:
            return 1                      # a test the map does not know yet
        return 0 if set(kernels) <= hw else 1
    items.sort(key=group)                 # stable


def load_golden(name):
    with open(os.path.join(GOLDEN, name), "r", encoding="utf-8") as f:
        return json.load(f)


@pytest.fixture(scope="session")
def golden_train():
    return load_golden("golden_train.json")


@pytest.fixture(scope="session")
def golden_cases():
    return load_golden("golden_cases.json")


@pytest.fixture(scope="session")
def golden_primitives():
    return load_golden("golden_primitives.json")


@pytest.fixture(scope="session")
def taylorswift():
    with open(os.path.join(GOLDEN, "taylorswift.txt"), "r", encoding="utf-8") as f:
        return f.read()
