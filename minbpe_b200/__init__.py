"""
minbpe_b200 — GPU-native (H100, sm_90a) byte-level BPE train/encode hot path behind the minbpe API.

    from minbpe_b200 import Tokenizer, BasicTokenizer, RegexTokenizer, GPT4Tokenizer

mirrors ``from minbpe import ...`` (reference minbpe/__init__.py:1-4).  The hot loops run in
hand-written sm_90a CUDA kernels reached through the C ABI in include/b200bpe.h.
"""
from .tokenizer import (  # noqa: F401
    GPT2_SPLIT_PATTERN,
    GPT4_SPLIT_PATTERN,
    BasicTokenizer,
    RegexTokenizer,
    Tokenizer,
    get_stats,
    merge,
)
from .gpt4 import GPT4Tokenizer  # noqa: F401,E402
