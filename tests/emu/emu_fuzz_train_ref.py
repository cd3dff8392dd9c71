#!/usr/bin/env python3
"""TEST INFRASTRUCTURE (BPE_LIB_PATH = the emulator build): BasicTokenizer / RegexTokenizer .train() of the product classes
(kernels on the emulator) against the UNMODIFIED reference classes on random small texts — tie-heavy alphabets, runs of
one character (the (a,a) path), texts that run out of pairs (both must raise ValueError and leave the tokenizer
untrained), both split patterns; merges, vocab, the ids of encode() and the saved .model / .vocab bytes must be identical.
What the reference computed for each round is stored in tests/golden/golden_fuzz_train.json (`--record` rewrites it from
the reference vendored into oracle/_ref by oracle/make_ref.py).

    BPE_LIB_PATH=tests/emu/_build/libb200bpe_emu.so python tests/emu/emu_fuzz_train_ref.py [rounds] [seed] [--record]
"""
import hashlib
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import minbpe_b200 as ours  # noqa: E402
from minbpe_b200.tokenizer import GPT2_SPLIT_PATTERN, GPT4_SPLIT_PATTERN  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_fuzz_train.json")


def sha(b):
    return hashlib.sha256(b).hexdigest()[:16]


def ids_sha(ids):
    return sha(np.asarray(ids, dtype="<i4").tobytes())


def vocab_sha(vocab):
    return sha(b"".join(i.to_bytes(4, "little") + len(v).to_bytes(4, "little") + v for i, v in sorted(vocab.items())))


def outcome(tok, text, vocab, tmp, name):
    """What one round produces: the merges, a digest of the vocab, of the ids of a probe text and of the saved files."""
    try:
        tok.train(text, vocab)
    except ValueError:
        return {"raises": True}
    probe = text[: 300] + " ab aab" + text[-50:]
    ids = tok.encode(probe)
    assert tok.decode(ids) == probe
    tok.save(os.path.join(tmp, name))
    files = {ext: sha(open(os.path.join(tmp, name + ext), "rb").read()) for ext in (".model", ".vocab")}
    return {"raises": False, "merges": [[a, b, i] for (a, b), i in tok.merges.items()], "vocab": vocab_sha(tok.vocab),
            "probe_n": len(ids), "probe_ids": ids_sha(ids), "files": files}


def random_text(rng):
    kind = rng.random()
    if kind < 0.3:
        alpha = list("ab")                                   # ties everywhere, long runs
    elif kind < 0.6:
        alpha = list("abc de'1\n")
    else:
        alpha = list("the quick brown fox é日 12 's 'll\t") + ["aaaa", "  ", "zzzzzz"]
    n = int(rng.choice([1, 2, 3, 5, 12, 40, 200, 1500]))
    return "".join(str(x) for x in rng.choice(alpha, size=n))


def main(rounds, seed, record):
    ref = None
    if record:
        from oracle import make_ref
        ref = make_ref.load()
        assert ref is not None, "oracle/_ref is not vendored (oracle/make_ref.py)"
        golden = {"rounds": rounds, "seed": seed, "cases": []}
    else:
        golden = json.load(open(GOLDEN))
        assert (golden["rounds"], golden["seed"]) == (rounds, seed), "tests/golden/golden_fuzz_train.json holds other rounds"
    rng = np.random.default_rng(seed)
    done = raised = 0
    tmp = tempfile.mkdtemp()
    for it in range(rounds):
        text = random_text(rng)
        vocab = 256 + int(rng.choice([0, 1, 2, 5, 20, 60]))
        which = int(rng.integers(0, 3))
        pat = GPT4_SPLIT_PATTERN if which == 1 else GPT2_SPLIT_PATTERN
        if record:
            r = ref.BasicTokenizer() if which == 0 else ref.RegexTokenizer(pat)
            golden["cases"].append(dict(outcome(r, text, vocab, tmp, "r"), text=sha(text.encode()), vocab_size=vocab, which=which))
            continue
        want = golden["cases"][it]
        assert (want["text"], want["vocab_size"], want["which"]) == (sha(text.encode()), vocab, which), f"round {it}: other inputs"
        o = ours.BasicTokenizer() if which == 0 else ours.RegexTokenizer(pat)
        got = outcome(o, text, vocab, tmp, "o")
        for k in ("raises", "merges", "vocab", "probe_n", "probe_ids", "files"):
            assert got.get(k) == want.get(k), (it, k, which, vocab, text)
        if got["raises"]:
            raised += 1
            assert not getattr(o, "merges", None) or o.merges == {}, "a failed train() must not leave merges behind"
        else:
            done += 1
    if record:
        with open(GOLDEN, "w") as f:
            json.dump(golden, f, separators=(",", ":"))
        print(f"recorded {rounds} rounds to {GOLDEN}")
        return 0
    print(f"emu fuzz train ok: {done} trained identically, {raised} ran out of pairs on both sides, of {rounds}")
    return 0


if __name__ == "__main__":
    record = "--record" in sys.argv
    argv = [a for a in sys.argv[1:] if a != "--record"]
    sys.exit(main(int(argv[0]) if argv else 100, int(argv[1]) if len(argv) > 1 else 5, record))
