"""CPU: the host side of RegexTokenizer.train(dedup=True) — count_chunks, the distinct chunks of a split text with their
counts in first-occurrence order — equals the oracle's orc_dedup_chunks under both split patterns and a custom one."""
import numpy as np
import pytest
import regex

import oracle
from minbpe_b200.tokenizer import GPT2_SPLIT_PATTERN, GPT4_SPLIT_PATTERN, count_chunks, split_text

PATTERNS = {"gpt4": GPT4_SPLIT_PATTERN, "gpt2": GPT2_SPLIT_PATTERN, "custom": r"\p{L}+|\s+|[^\s\p{L}]+"}


def _random_text(seed, n):
    rng = np.random.default_rng(seed)
    alphabet = list("aab  bc\n\t'sé中😀1234.,!?") + ["the ", "The ", "  ", "'ll", "\r\n"]
    return "".join(alphabet[i] for i in rng.integers(0, len(alphabet), n))


@pytest.mark.parametrize("pattern", sorted(PATTERNS))
def test_count_chunks_equals_the_oracle(pattern, taylorswift):
    pat = regex.compile(PATTERNS[pattern])
    for text in [taylorswift, "", "x", "aaaa"] + [_random_text(s, 3000) for s in range(5)]:
        data, offs = split_text(pat, text)
        ub, uo, uw = count_chunks(data, offs)
        ob, oo, ow = oracle.c_dedup_chunks(data, offs)
        assert ub == ob.tobytes(), text[:40]
        assert np.array_equal(uo, oo.astype(np.uint64)) and np.array_equal(uw, ow.astype(np.uint64)), text[:40]
        assert int(uw.sum()) == len(offs)
