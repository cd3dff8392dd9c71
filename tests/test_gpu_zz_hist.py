"""GPU: the packed dense byte-pair histogram (k_hist_dense_packed, b200bpe.cu hist_dense).  Forced on
(BPE_OPT_HIST_KERNEL = 1) it must train exactly like the oracle; with BPE_OPT_HIST_KERNEL = 0 the library decides at the
first large stream — both kernels run, the 65,536 counters are compared on the device and the launches timed — and
whatever it decides, results do not change.  (Default: 2, k_hist_dense.)"""
import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu


def test_packed_histogram_forced():
    from minbpe_b200 import engine as E
    from minbpe_b200.synth import generate
    eng = E.Engine(0)
    eng.set_option(E.OPT_HIST_KERNEL, 1)
    raw = generate(1337, 3 << 20)
    for n, merges in ((3 << 20, 6), (70001, 4), (513, 3), (2, 1)):
        eng.load_stream(raw[:n], None)                      # one chunk: every adjacent pair counts
        p, c, d = eng.train(merges)
        assert eng.timing()["hist_kernel"] == 1
        w = oracle.c_train(raw[:n].astype(np.int32), None, merges)
        assert d == w[2] and np.array_equal(p, w[0]) and np.array_equal(c, w[1]), n
    with pytest.raises(E.EngineError):
        eng.set_option(E.OPT_HIST_KERNEL, 3)
    eng.close()


def test_histogram_choice_is_made_on_a_large_stream_and_is_harmless():
    from minbpe_b200 import engine as E
    from minbpe_b200.synth import generate
    eng = E.Engine(0)
    eng.set_option(E.OPT_HIST_KERNEL, 0)                    # decide at the first large stream (the default is k_hist_dense)
    raw = generate(1338, 9 << 20)
    eng.load_stream(raw[:100000], None)
    eng.train(3)
    assert eng.timing()["hist_kernel"] == 0                 # too small to say anything about speed: k_hist_dense, undecided
    eng.load_stream(raw, None)                              # 9 Mi tokens: cross-check + timing
    p, c, d = eng.train(5)
    chosen = eng.timing()["hist_kernel"]
    assert chosen in (1, 2)
    w = oracle.c_train(raw.astype(np.int32), None, 5)
    assert np.array_equal(p, w[0]) and np.array_equal(c, w[1])
    eng.load_stream(raw[:200000], None)                     # decided: the same kernel from now on, whatever the size
    p, c, d = eng.train(4)
    assert eng.timing()["hist_kernel"] == chosen
    w = oracle.c_train(raw[:200000].astype(np.int32), None, 4)
    assert np.array_equal(p, w[0]) and np.array_equal(c, w[1])
    print("histogram kernel chosen:", {1: "k_hist_dense_packed", 2: "k_hist_dense"}[chosen])
    eng.close()
