"""CPU: device-memory ownership of the host side on the SIMT emulator (tests/emu/emu_ownership.py, as tests/test_emu_docs.py
runs the emulator): create + every family + destroy leaves no allocation or event live; a cudaMalloc that fails at any
point of a family is reported as BPE_ERR_CUDA, the handle then gives the clean result and releases everything; a larger
load_stream never holds the old and the new stream buffers together.  Once against the plain build and once against the
UBSan build (alignment, shift counts, array bounds)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
CASES = ["released", "peak", "create", "train", "train_filter", "ids", "replay", "encode_short", "encode_long", "encode_text",
         "encode_special", "decode", "session", "weighted", "weighted_dedup"]


@pytest.fixture(scope="module", params=["plain", "ubsan"])
def emu_lib(request):
    if request.param == "plain":
        sys.path.insert(0, EMU)
        import build_emu
        return build_emu.build(), {}
    out = subprocess.run([sys.executable, os.path.join(EMU, "build_emu.py"), "--force"], cwd=ROOT, check=True, text=True,
                         stdout=subprocess.PIPE, env=dict(os.environ, EMU_SANITIZE="1")).stdout
    lib = out.strip().splitlines()[-1]
    assert lib.endswith("_ubsan.so")
    ubsan = subprocess.run(["g++", "-print-file-name=libubsan.so"], check=True, text=True, stdout=subprocess.PIPE).stdout.strip()
    return lib, {"LD_PRELOAD": ubsan}


@pytest.mark.parametrize("case", CASES)
def test_emu_ownership(emu_lib, case):
    lib, extra = emu_lib
    env = dict(os.environ, BPE_LIB_PATH=lib, EMU_SMS="2", PYTHONDONTWRITEBYTECODE="1", **extra)
    p = subprocess.run([sys.executable, os.path.join(EMU, "emu_ownership.py"), case], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0 and p.stdout.rstrip().endswith("ok"), p.stdout[-6000:]
