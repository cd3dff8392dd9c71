"""
Unicode class tables for the device-side splitter (include/b200bpe.h bpe_gpt4_tables, bpe_o200k_table),
enumerated from the INSTALLED `regex` module so that the device split agrees with
`regex.findall(GPT4_SPLIT_PATTERN, ...)` of this very installation (its tables are newer than
`unicodedata`, SURVEY.md §0.3).  Cached next to the library (csrc/gpt4_tables.npz, csrc/o200k_tables.npz).
"""
import os

import numpy as np
import regex

_HERE = os.path.dirname(os.path.abspath(__file__))
_CACHE = os.path.join(_HERE, "csrc", "gpt4_tables.npz")
_CACHE_O200K = os.path.join(_HERE, "csrc", "o200k_tables.npz")
C_L, C_N, C_NL, C_SP, C_AP, C_O = 0, 1, 2, 3, 4, 5
# case classes of the o200k pattern (split_logic.h SC_CU ..): 0 = none of them
K_NONE, K_UPPER, K_LOWER, K_BOTH, K_MARK = 0, 1, 2, 3, 4
_tables = None
_o200k = None


def _enumerate():
    cls = np.full(0x110000, C_O, dtype=np.uint8)
    pl, pn, ps = regex.compile(r"\p{L}"), regex.compile(r"\p{N}"), regex.compile(r"\s")
    for cp in range(0x110000):
        if 0xD800 <= cp <= 0xDFFF:
            continue
        ch = chr(cp)
        if pl.match(ch):
            cls[cp] = C_L
        elif pn.match(ch):
            cls[cp] = C_N
        elif ps.match(ch):
            cls[cp] = C_SP
    cls[0x0D] = cls[0x0A] = C_NL
    cls[0x27] = C_AP
    contr = np.zeros(0x3000, dtype=np.uint8)
    groups = (("[sdmt]", 1), ("l", 2), ("v", 4), ("e", 8), ("r", 16))
    pats = [(regex.compile("(?i:%s)" % g), bit) for g, bit in groups]
    for cp in range(0x3000):
        ch = chr(cp)
        for p, bit in pats:
            if p.fullmatch(ch):
                contr[cp] |= bit
    return cls, contr


def tables():
    """(cls uint8[0x110000], contr uint8[0x3000]) for bpe_gpt4_tables."""
    global _tables
    if _tables is None:
        ver = regex.__version__
        if os.path.exists(_CACHE):
            try:
                z = np.load(_CACHE)
                if str(z["regex_version"]) == ver:
                    _tables = (np.ascontiguousarray(z["cls"]), np.ascontiguousarray(z["contr"]))
            except Exception:  # noqa: BLE001
                _tables = None
        if _tables is None:
            cls, contr = _enumerate()
            try:
                np.savez_compressed(_CACHE, cls=cls, contr=contr, regex_version=ver)
            except OSError:
                pass
            _tables = (cls, contr)
    return _tables


def _enumerate_o200k():
    cps = np.array([cp for cp in range(0x110000) if not 0xD800 <= cp <= 0xDFFF], dtype=np.int64)
    text = "".join(map(chr, cps.tolist()))
    case = np.zeros(0x110000, dtype=np.uint8)
    for pat, k in ((r"[\p{Lu}\p{Lt}]", K_UPPER), (r"\p{Ll}", K_LOWER), (r"[\p{Lm}\p{Lo}]", K_BOTH), (r"\p{M}", K_MARK)):
        at = np.array([m.start() for m in regex.finditer(pat, text)], dtype=np.int64)
        case[cps[at]] = k
    return case


def o200k_table():
    """case uint8[0x110000] for bpe_o200k_table: the o200k pattern's letter classes (K_UPPER = Lu/Lt, K_LOWER = Ll,
    K_BOTH = Lm/Lo, K_MARK = M, K_NONE = everything else)."""
    global _o200k
    if _o200k is None:
        ver = regex.__version__
        if os.path.exists(_CACHE_O200K):
            try:
                z = np.load(_CACHE_O200K)
                if str(z["regex_version"]) == ver:
                    _o200k = np.ascontiguousarray(z["case"])
            except Exception:  # noqa: BLE001
                _o200k = None
        if _o200k is None:
            _o200k = _enumerate_o200k()
            try:
                np.savez_compressed(_CACHE_O200K, case=_o200k, regex_version=ver)
            except OSError:
                pass
    return _o200k
