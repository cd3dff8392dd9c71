"""CPU: the checks of the reference's own test file (karpathy/minbpe tests/test_tokenizer.py) against minbpe_b200, with
what the reference computed stored under tests/golden/ (golden_reference_suite.json, golden_train.json): encode/decode
identity of the untrained tokenizers, the Wikipedia known-answer test, and save/load with and without special tokens.
No GPU here, so the library under the classes is the CPU SIMT emulator build of the kernel sources (tests/emu/), in a
subprocess that runs this file as a script.  The GPT4Tokenizer checks of that file need tiktoken's cl100k_base (a
download) and are not part of it.

    python tests/test_reference_suite.py --record <karpathy/minbpe checkout>    # rewrite golden_reference_suite.json
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SUITE = os.path.join(GOLDEN, "golden_reference_suite.json")


def ids_sha(ids):
    import numpy as np
    return hashlib.sha256(np.asarray(ids, dtype="<i4").tobytes()).hexdigest()


def _texts(suite):
    """The fixture strings of the reference's test file; "FILE:taylorswift.txt" stands for the corpus."""
    taylor = open(os.path.join(GOLDEN, "taylorswift.txt"), encoding="utf-8").read()
    return [taylor if t == "FILE:taylorswift.txt" else t for t in suite["test_strings"]]


def record(ref):
    sys.path.insert(0, ref)
    from minbpe import BasicTokenizer, RegexTokenizer
    from tests.test_tokenizer import test_strings
    suite = {"test_strings": list(test_strings), "identity": {}}
    for name, cls in (("basic", BasicTokenizer), ("regex", RegexTokenizer)):
        suite["identity"][name] = [{"n_ids": len(ids), "ids_sha256": ids_sha(ids)}
                                   for ids in (cls().encode(t) for t in _texts(suite))]
    with open(SUITE, "w", encoding="utf-8") as f:
        json.dump(suite, f, indent=0, ensure_ascii=True)


def check():
    """Runs with BPE_LIB_PATH = the emulator build (see the test below)."""
    sys.path.insert(0, ROOT)
    from minbpe_b200 import BasicTokenizer, RegexTokenizer
    suite = json.load(open(SUITE, encoding="utf-8"))
    train = json.load(open(os.path.join(GOLDEN, "golden_train.json"), encoding="utf-8"))
    n = 0
    # encode/decode identity (test_tokenizer.py:51-59), untrained tokenizers: the reference's ids
    for name, cls in (("basic", BasicTokenizer), ("regex", RegexTokenizer)):
        for text, want in zip(_texts(suite), suite["identity"][name]):
            tok = cls()
            ids = tok.encode(text)
            assert (len(ids), ids_sha(ids)) == (want["n_ids"], want["ids_sha256"]), (name, text[:40])
            assert tok.decode(ids) == text
            n += 1
    # Wikipedia example (test_tokenizer.py:79-107): the reference's merges and ids
    for name, cls in (("basic", BasicTokenizer), ("regex", RegexTokenizer)):
        want = train[f"wikipedia_{name}"]
        tok = cls()
        tok.train("aaabdaaabac", 256 + 3)
        ids = tok.encode("aaabdaaabac")
        assert ids == want["ids"] == [258, 100, 258, 97, 99]
        assert [list(p) for p in tok.merges] == want["merges"]
        assert tok.decode(tok.encode("aaabdaaabac")) == "aaabdaaabac"
        n += 1
    # save/load with and without special tokens (test_tokenizer.py:109-132): the reference's merges, ids and .model file
    llama = open(os.path.join(GOLDEN, "llama_text.txt"), encoding="utf-8").read()
    want = train["llama_regex_320_specials"]
    for specials in ({}, want["specials"]):
        tok = RegexTokenizer()
        tok.train(llama, 256 + 64)
        assert [list(p) for p in tok.merges] == want["merges"]
        tok.register_special_tokens(specials)
        ids = tok.encode(llama, "all")
        assert ids == (want["ids_all"] if specials else want["ids_none"])
        assert tok.decode(ids) == llama
        with tempfile.TemporaryDirectory() as d:
            prefix = os.path.join(d, "test_tokenizer_tmp")
            tok.save(prefix)
            if specials:
                assert open(prefix + ".model", encoding="utf-8").read() == want["model_text"]
            tok = RegexTokenizer()
            tok.load(prefix + ".model")
        assert tok.decode(ids) == llama
        assert tok.decode(tok.encode(llama, "all")) == llama
        assert tok.encode(llama, "all") == ids
        n += 1
    print(f"reference suite ok: {n} checks")


def test_reference_suite_against_reference_goldens(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    lib = build_emu.build()
    env = dict(os.environ, BPE_LIB_PATH=lib, PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTEST_CURRENT_TEST", None)
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "reference suite ok: 12 checks" in r.stdout, r.stdout[-1000:]


if __name__ == "__main__":
    record(sys.argv[2]) if sys.argv[1:2] == ["--record"] else check()
