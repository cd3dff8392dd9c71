"""GPU: the statistics delta of k_merge_seg on both sides of its shared-counter threshold.  A pass whose NK·(2V+1) delta
indices fit in MS_DELTA_WORDS gives every index its own shared counter; a larger one folds them through the hashed
cache.  One training run, split into bpe_train calls whose delta layout V (BPE_OPT_VOCAB_CAP) puts batched passes on
either side, must still give the oracle's merges, counts, stream and pair table, and the passes the host model predicts
(tests/batch_model.py)."""
import os
import re

import numpy as np
import pytest
import regex

import oracle
from batch_model import ROOT, partition, stats, table_dict

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpora, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")


def delta_words():
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", "k_merge_seg.cuh")) as f:
        return int(re.search(r"#define MS_DELTA_WORDS (\d+)", f.read()).group(1))


def test_direct_and_hashed_delta(taylorswift):
    from minbpe_b200 import engine as E
    words = delta_words()
    text = taylorswift[: 60000] if SMALL else taylorswift
    data, offs = oracle.split_to_stream(text, GPT4)
    ids = np.asarray(data, dtype=np.int32)
    total = 150 if SMALL else 300
    calls = [(100, 0), (25, 600), (total - 125, 4000)]   # (merges, BPE_OPT_VOCAB_CAP)
    wp, wc, _, fin = oracle.c_train(ids, offs, total, want_final=True)

    eng = E.Engine(0)
    eng.set_option(E.OPT_BATCH, 8)
    eng.load_stream(ids.astype(np.uint8), offs)
    cur, cur_offs, fi, sides = ids, offs, 256, set()
    for n, cap in calls:
        m = partition(cur, cur_offs, n, first_idx=fi)
        # bpe_train's delta layout: V = max(first_idx + merges, max id + 1, BPE_OPT_VOCAB_CAP); every id is below first_idx
        assert int(cur.max()) < fi
        V = max(fi + n, cap)
        sides |= {(nk > 1, nk * (2 * V + 1) <= words) for nk in m.sizes}
        eng.set_option(E.OPT_VOCAB_CAP, cap)
        p, c, d = eng.train(n, first_idx=fi)
        assert d == n and np.array_equal(p, wp[fi - 256: fi - 256 + n]) and np.array_equal(c, wc[fi - 256: fi - 256 + n])
        assert eng.timing()["tokens_in"] == m.tokens_in, (n, cap, m.sizes)
        cur, cur_offs, fi = m.final, m.final_offs, fi + n
    # batched passes (and one-member passes) ran with direct counters and with the hashed cache
    assert sides == {(True, True), (True, False), (False, True), (False, False)}, sides
    assert np.array_equal(eng.read_stream(), fin)
    st = np.zeros(len(fin), dtype=bool)
    st[cur_offs.astype(np.int64)] = True
    assert eng.debug_table() == table_dict(*stats(fin, st))
    eng.close()
