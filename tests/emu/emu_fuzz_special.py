#!/usr/bin/env python3
"""TEST INFRASTRUCTURE (BPE_LIB_PATH = the emulator build): RegexTokenizer.encode(text, allowed_special=...) with the
special tokens found, the parts split and everything encoded on the device (k_special.cuh, split_logic.h WITH_B,
k_encode2.cuh) against the UNMODIFIED reference class on random texts: specials that are prefixes of one another,
adjacent and overlapping occurrences, specials at either end of the text, white space / letters / digits / apostrophes on
both sides (the split of a part must behave as on a text of its own), both split patterns, subsets as `allowed_special`,
several pieces per call.  The reference's merges and what it returned for each round are stored in
tests/golden/golden_fuzz_special.json (`--record` rewrites it from the reference vendored into oracle/_ref by
oracle/make_ref.py).

    BPE_LIB_PATH=tests/emu/_build/libb200bpe_emu.so python tests/emu/emu_fuzz_special.py [rounds] [seed] [--record]
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from minbpe_b200 import RegexTokenizer  # noqa: E402
from minbpe_b200 import engine as E  # noqa: E402
from minbpe_b200.tokenizer import GPT2_SPLIT_PATTERN, GPT4_SPLIT_PATTERN  # noqa: E402

POOL = ["<|endoftext|>", "<|end|>", "<|endof", "<|a|>", "<|a|><|b|>", "<|b|>", "<s>", "</s>", "<s", "[SEP]", "[S", " <pad>", "<|é|>", "'s<", "12", "\n\n<|x|>"]
FILL = list("abcde  é1!'\n\t") + ["日", " the", "'ll", "  ", "\r\n", "42"]
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_fuzz_special.json")
PATTERNS = {"gpt4": GPT4_SPLIT_PATTERN, "gpt2": GPT2_SPLIT_PATTERN}


def sha(b):
    return hashlib.sha256(b).hexdigest()[:16]


def ids_sha(ids):
    return sha(np.asarray(ids, dtype="<i4").tobytes())


def random_case(rng):
    k = int(rng.integers(1, 6))
    toks = [str(x) for x in rng.choice(POOL, size=k, replace=False)]
    special = {t: 1000 + i for i, t in enumerate(toks)}
    parts = []
    for _ in range(int(rng.integers(1, 60))):
        r = rng.random()
        if r < 0.35:
            parts.append(str(rng.choice(toks)))
        elif r < 0.45:
            t = str(rng.choice(toks))
            parts.append(t[: int(rng.integers(1, len(t) + 1))])          # a truncated special: must stay ordinary text
        else:
            parts.append("".join(str(x) for x in rng.choice(FILL, size=int(rng.integers(1, 12)))))
    return special, "".join(parts)


def main(rounds, seed, record):
    train_text = open(os.path.join(ROOT, "tests", "golden", "taylorswift.txt"), encoding="utf-8").read()[:60000]
    toks = {}
    if record:
        from oracle import make_ref
        ref = make_ref.load()
        assert ref is not None, "oracle/_ref is not vendored (oracle/make_ref.py)"
        golden = {"rounds": rounds, "seed": seed, "merges": {}, "cases": []}
        for name, pat in PATTERNS.items():
            r = ref.RegexTokenizer(pat)
            r.train(train_text[:20000], 256 + 120)
            golden["merges"][name] = [[a, b, i] for (a, b), i in r.merges.items()]
            toks[pat] = r
    else:
        golden = json.load(open(GOLDEN))
        assert (golden["rounds"], golden["seed"]) == (rounds, seed), "tests/golden/golden_fuzz_special.json holds other rounds"
        for name, pat in PATTERNS.items():
            o = RegexTokenizer(pat)
            o.merges = {(a, b): i for a, b, i in golden["merges"][name]}
            o.vocab = o._build_vocab()
            o.DEVICE_SPLIT_MIN_BYTES = 0          # every text takes the device path, however short
            toks[pat] = o
    rng = np.random.default_rng(seed)
    n_dev = 0
    for it in range(rounds):
        special, text = random_case(rng)
        if rng.random() < 0.2:
            text = text + " " + train_text[: int(rng.integers(100, 5000))] + text
        pat = GPT4_SPLIT_PATTERN if rng.random() < 0.6 else GPT2_SPLIT_PATTERN
        tok = toks[pat]
        tok.register_special_tokens(special)
        allowed = "all" if rng.random() < 0.7 else set(list(special)[: int(rng.integers(0, len(special) + 1))])
        piece = int(rng.choice([0, 0, 0, 4096]))
        inputs = sha(json.dumps([special, text, pat == GPT4_SPLIT_PATTERN, sorted(allowed) if isinstance(allowed, set) else allowed,
                                 piece]).encode())
        if record:
            want = tok.encode(text, allowed_special=allowed)
            golden["cases"].append({"inputs": inputs, "n_ids": len(want), "ids": ids_sha(want),
                                    "decoded": sha(tok.decode(want).encode("utf-8"))})
            continue
        want = golden["cases"][it]
        assert want["inputs"] == inputs, f"round {it}: other inputs"
        tok.engine.set_option(E.OPT_SPLIT_PIECE, piece)
        try:
            try:
                got = tok.encode(text, allowed_special=allowed)
            except E.EngineError as ex:       # a tiny piece size may find no letter+space cut: a clean error, not a wrong answer
                assert "cut point" in str(ex), ex
                continue
        finally:
            tok.engine.set_option(E.OPT_SPLIT_PIECE, 0)
        assert (len(got), ids_sha(got)) == (want["n_ids"], want["ids"]), (it, pat == GPT4_SPLIT_PATTERN, special, allowed, text)
        assert sha(tok.decode(got).encode("utf-8")) == want["decoded"]
        n_dev += 1
    if record:
        with open(GOLDEN, "w") as f:
            json.dump(golden, f, separators=(",", ":"))
        print(f"recorded {rounds} rounds to {GOLDEN}")
        return 0
    print(f"emu fuzz special ok: {n_dev} of {rounds} rounds compared with the reference class")
    return 0


if __name__ == "__main__":
    record = "--record" in sys.argv
    argv = [a for a in sys.argv[1:] if a != "--record"]
    sys.exit(main(int(argv[0]) if argv else 100, int(argv[1]) if len(argv) > 1 else 5, record))
