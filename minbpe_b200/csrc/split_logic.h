// split_logic.h — the GPT-4 split pattern (regex.py:19) as pure functions of LOCAL data: the scan
// element / combine operators of six segmented scans over class runs, and the rule "does a chunk
// start at this character?" written on the scan results at a byte and at its predecessor plus a
// few neighbouring bytes.  Specification and derivation: oracle/split_rules_local.py, DESIGN.md §9.
//
// Plain C++ on purpose: the CUDA kernels (k_split.cuh) and the CPU harness that pins this file
// against the `regex` module (oracle/split_harness.cpp, tests/test_split_rules.py) compile the same
// functions.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SPL_HD __host__ __device__ __forceinline__
#else
#define SPL_HD inline
#endif

// character classes (one per code point; table enumerated from the `regex` module)
#define SC_L 0u    // \p{L}
#define SC_N 1u    // \p{N}
#define SC_NL 2u   // \r \n
#define SC_SP 3u   // other \s
#define SC_AP 4u   // apostrophe
#define SC_O 5u    // everything else
#define SC_B 6u    // bytes of a special-token occurrence (regex.py:152-163): the text on either side is split on its own, so such
                   // a byte ends the runs around it and counts as "end of text" / "start of text" for its neighbours.  Only the
                   // WITH_B instantiations of the functions below know this class; the plain GPT-4 split never produces it.
#define SM_CLS 7u
#define SM_START 8u     // meta bit: first byte of a UTF-8 sequence
#define SM_SPEC 16u     // meta bit: byte of a special-token occurrence in a split buffer of documents (k_special_meta<true>), which
                        // tells it apart from a document gap (also SC_B); the rule below never reads it
#define SPL_PK_NONE 7u  // "kind of the character in front of the run" at the start of the text

// run kind: letters, digits, whitespace (SP or NL), other (O or apostrophe)
SPL_HD uint32_t spl_kind(uint32_t cls) { return cls == SC_NL ? SC_SP : (cls == SC_AP ? SC_O : cls); }

// ---- UTF-8 ----------------------------------------------------------------------------------
template <class Bytes>
SPL_HD uint32_t spl_utf8_decode(const Bytes &b, uint64_t i, uint64_t n) {
    const uint32_t c0 = b(i);
    if (c0 < 0x80) return c0;
    const uint32_t c1 = (i + 1 < n ? b(i + 1) : 0u) & 0x3fu;
    if (c0 < 0xE0) return ((c0 & 0x1fu) << 6) | c1;
    const uint32_t c2 = (i + 2 < n ? b(i + 2) : 0u) & 0x3fu;
    if (c0 < 0xF0) return ((c0 & 0x0fu) << 12) | (c1 << 6) | c2;
    const uint32_t c3 = (i + 3 < n ? b(i + 3) : 0u) & 0x3fu;
    return ((c0 & 0x07u) << 18) | (c1 << 12) | (c2 << 6) | c3;
}
SPL_HD uint32_t spl_utf8_len(uint32_t cp) { return cp < 0x80 ? 1u : cp < 0x800 ? 2u : cp < 0x10000 ? 3u : 4u; }
// first byte of the character that byte i belongs to
template <class Bytes>
SPL_HD uint64_t spl_char_start(const Bytes &b, uint64_t i) {
    while (i > 0 && (b(i) & 0xC0u) == 0x80u) --i;
    return i;
}
// meta of byte i = class of its character | SM_START on the character's first byte
template <class Bytes>
SPL_HD uint32_t spl_meta_of(const Bytes &b, uint64_t i, uint64_t n, const uint8_t *cls_table) {
    const bool start = (b(i) & 0xC0u) != 0x80u;
    const uint64_t s = start ? i : spl_char_start(b, i);
    uint32_t cp = spl_utf8_decode(b, s, n);
    if (cp > 0x10ffffu) cp = 0xfffd;
    return (uint32_t)cls_table[cp] | (start ? SM_START : 0u);
}

// ---- forward segmented scan (segments = runs; reset at a run's first byte) --------------------
//   since  character starts of the run up to and including this byte
//   pk     kind of the byte in front of the run (SPL_PK_NONE at the start of the text)
//   lead   every byte of the run up to and including this one belongs to a newline
struct SplFwd {
    uint32_t since;
    uint32_t bits;   // pk (3 bits) | lead << 3 | first << 4
};
#define SPL_F_PK 7u
#define SPL_F_LEAD 8u
#define SPL_F_FIRST 16u
SPL_HD SplFwd spl_fwd_identity() { SplFwd r; r.since = 0; r.bits = SPL_F_LEAD; return r; }
// a = everything to the left, b = what follows it
SPL_HD SplFwd spl_fwd_combine(SplFwd a, SplFwd b) {
    if (b.bits & SPL_F_FIRST) return b;
    SplFwd r;
    r.since = a.since + b.since;
    r.bits = (a.bits & (SPL_F_PK | SPL_F_FIRST)) | (a.bits & b.bits & SPL_F_LEAD);
    return r;
}
// element of byte i: m = its meta, mprev = meta of byte i-1 (ignored for i == 0)
SPL_HD SplFwd spl_fwd_elem(uint64_t i, uint32_t m, uint32_t mprev) {
    const uint32_t cls = m & SM_CLS;
    const bool first = (i == 0) || spl_kind(mprev & SM_CLS) != spl_kind(cls);
    SplFwd r;
    r.since = (m & SM_START) ? 1u : 0u;
    r.bits = (cls == SC_NL ? SPL_F_LEAD : 0u);
    if (first) r.bits |= SPL_F_FIRST | (i == 0 ? SPL_PK_NONE : spl_kind(mprev & SM_CLS));
    return r;
}

// ---- backward segmented scan (reset at a run's last byte) -------------------------------------
//   toend  character starts of the run from this byte to the end of the run
//   nlah   some byte of the run at or after this one belongs to a newline
//   atend  the run ends at the end of the text
struct SplBwd {
    uint32_t toend;
    uint32_t bits;   // nlah | atend << 1 | last << 2
};
#define SPL_B_NLAH 1u
#define SPL_B_ATEND 2u
#define SPL_B_LAST 4u
SPL_HD SplBwd spl_bwd_identity() { SplBwd r; r.toend = 0; r.bits = 0; return r; }
// a = what comes first in the text, b = everything to the right of it
SPL_HD SplBwd spl_bwd_combine(SplBwd a, SplBwd b) {
    if (a.bits & SPL_B_LAST) return a;
    SplBwd r;
    r.toend = a.toend + b.toend;
    r.bits = (b.bits & (SPL_B_ATEND | SPL_B_LAST)) | ((a.bits | b.bits) & SPL_B_NLAH);
    return r;
}
// element of byte i: mnext = meta of byte i+1 (ignored for i + 1 == n)
template <bool WITH_B = false>
SPL_HD SplBwd spl_bwd_elem(uint64_t i, uint64_t n, uint32_t m, uint32_t mnext) {
    const uint32_t cls = m & SM_CLS;
    const bool last = (i + 1 == n) || spl_kind(mnext & SM_CLS) != spl_kind(cls);
    const bool text_ends = (i + 1 == n) || (WITH_B && (mnext & SM_CLS) == SC_B);
    SplBwd r;
    r.toend = (m & SM_START) ? 1u : 0u;
    r.bits = (cls == SC_NL ? SPL_B_NLAH : 0u);
    if (last) r.bits |= SPL_B_LAST | (text_ends ? SPL_B_ATEND : 0u);
    return r;
}

// ---- contractions ---------------------------------------------------------------------------
// contr[cp] (cp < 0x3000): bit 0 = matches (?i:[sdmt]), 1 = (?i:l), 2 = (?i:v), 3 = (?i:e), 4 = (?i:r)
SPL_HD uint32_t spl_contr_bits(const uint8_t *contr, uint32_t cp) { return cp < 0x3000u ? contr[cp] : 0u; }
// length in characters (2 or 3) of the contraction whose apostrophe is followed by the characters at byte s, or 0
template <class Bytes>
SPL_HD uint32_t spl_contraction_len(const Bytes &b, uint64_t n, const uint8_t *contr, uint64_t s) {
    if (s >= n) return 0;
    const uint32_t c1 = spl_utf8_decode(b, s, n);
    const uint32_t b1 = spl_contr_bits(contr, c1);
    if (b1 & 1u) return 2;
    const uint64_t s2 = s + spl_utf8_len(c1);
    if (s2 >= n) return 0;
    const uint32_t b2 = spl_contr_bits(contr, spl_utf8_decode(b, s2, n));
    if (((b1 & 2u) && (b2 & 2u)) || ((b1 & 4u) && (b2 & 8u)) || ((b1 & 16u) && (b2 & 8u))) return 3;
    return 0;
}

// byte x is a U+0020 of the text (with boundaries: not a 0x20 inside a special token)
template <bool WITH_B, class Bytes, class Meta>
SPL_HD bool spl_is_space20(const Bytes &b, const Meta &meta, uint64_t x) {
    return b(x) == 0x20u && (!WITH_B || (meta(x) & SM_CLS) == SC_SP);
}

// the character [p, pend) is a one-character Oish run that itself starts a match (no U+0020 in front)
template <bool WITH_B = false, class Bytes, class Meta>
SPL_HD bool spl_single_oish_start(const Bytes &b, const Meta &meta, uint64_t n, uint64_t p, uint64_t pend) {
    if (spl_kind(meta(p) & SM_CLS) != SC_O) return false;
    if (p > 0 && spl_kind(meta(p - 1) & SM_CLS) == SC_O) return false;
    if (pend < n && spl_kind(meta(pend) & SM_CLS) == SC_O) return false;
    return p == 0 || !spl_is_space20<WITH_B>(b, meta, p - 1);
}

// ---- the rule -------------------------------------------------------------------------------
// Does a chunk start at byte i?  i must be the first byte of a character.  f / g = inclusive forward /
// backward scan values at byte i, fprev = forward value at byte i-1 (anything for i == 0).
// Reads b() and meta() at most 12 bytes before and 8 bytes after i.
// WITH_B: bytes of class SC_B separate independently split texts (see SC_B); the caller overrides the answer for those
// bytes themselves and for the byte that follows them.
template <bool WITH_B = false, class Bytes, class Meta>
SPL_HD bool spl_chunk_start(uint64_t i, uint64_t n, SplFwd f, SplFwd fprev, SplBwd g, const Bytes &b, const Meta &meta,
                            const uint8_t *contr) {
    if (i == 0) return true;
    const uint32_t cls = meta(i) & SM_CLS, kind = spl_kind(cls);
    if (WITH_B && cls == SC_B) return false;
    const uint32_t before = f.since - 1u;            // characters of the run in front of this one
    if (kind == SC_N) return before % 3u == 0u;      // \p{N}{1,3}: groups of three from the start of the run
    if (kind == SC_O) return before == 0u && !spl_is_space20<WITH_B>(b, meta, i - 1);   // with a space in front, the space starts the chunk
    if (kind == SC_SP) {
        const bool prev_oish = (f.bits & SPL_F_PK) == SC_O;       // " ?[^\s\p{L}\p{N}]++[\r\n]*" took the leading newlines
        const bool is_nl = cls == SC_NL;
        const bool in_run = before > 0u;
        const bool lead_prev = in_run && (fprev.bits & SPL_F_LEAD);
        const bool is_w2s = prev_oish ? (!is_nl && (!in_run || lead_prev)) : !in_run;
        const bool prev_is_nl = in_run && (meta(i - 1) & SM_CLS) == SC_NL;
        const bool nlah = (g.bits & SPL_B_NLAH) != 0, atend = (g.bits & SPL_B_ATEND) != 0;
        const bool is_w3s = !nlah && ((prev_is_nl && !(prev_oish && lead_prev)) || is_w2s);
        const bool rule_a = is_w2s && nlah;                        // \s*[\r\n]
        const bool rule_b = is_w3s && (atend || g.toend >= 2u);    // \s+(?!\S)
        const bool rule_c = g.toend == 1u && !atend && !is_nl;     // the last space joins what follows
        return rule_a || rule_b || rule_c;
    }
    // letters
    if (before == 0u) {
        const uint64_t p = spl_char_start(b, i - 1);
        if ((meta(p) & SM_CLS) == SC_SP) return false;             // absorbed as the optional prefix
        return !spl_single_oish_start<WITH_B>(b, meta, n, p, i);
    }
    if (before <= 2u) {   // second or third letter of a run that follows a contraction apostrophe: "'s|foo", "'ll|ama"
        uint64_t s = i;
        for (uint32_t c = 0; c < before; ++c) s = spl_char_start(b, s - 1);
        if (s >= 1 && b(s - 1) == 0x27u && spl_single_oish_start<WITH_B>(b, meta, n, s - 1, s)) {
            const uint32_t clen = spl_contraction_len(b, n, contr, s);
            return clen != 0u && before == clen - 1u;
        }
    }
    return false;
}

// ---- the GPT-2 pattern (regex.py:18) on the same scans ------------------------------------------------------------
//   '(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+
// Simpler than the GPT-4 one: a run of letters, of digits or of "Oish" characters is one chunk, with a single U+0020 in
// front joining it; a whitespace run is one chunk, except that its last character is split off when something follows
// (it joins the next chunk if it is U+0020, stands alone otherwise); contractions are ASCII and case-sensitive, and only
// tried where the apostrophe is a match start (a one-character Oish run without a space in front).
template <class Bytes>
SPL_HD uint32_t spl_contraction_len_gpt2(const Bytes &b, uint64_t n, uint64_t s) {
    if (s >= n) return 0;
    const uint32_t c1 = b(s);
    if (c1 == 's' || c1 == 'd' || c1 == 'm' || c1 == 't') return 2;
    if (s + 1 >= n) return 0;
    const uint32_t c2 = b(s + 1);
    if ((c1 == 'l' && c2 == 'l') || (c1 == 'v' && c2 == 'e') || (c1 == 'r' && c2 == 'e')) return 3;
    return 0;
}

template <bool WITH_B = false, class Bytes, class Meta>
SPL_HD bool spl_chunk_start_gpt2(uint64_t i, uint64_t n, SplFwd f, SplBwd g, const Bytes &b, const Meta &meta) {
    if (i == 0) return true;
    const uint32_t cls = meta(i) & SM_CLS, kind = spl_kind(cls);
    if (WITH_B && cls == SC_B) return false;
    const uint32_t before = f.since - 1u;            // characters of the run in front of this one
    if (kind == SC_SP) {
        if (before == 0u) return true;                                   // \s+(?!\S) / \s+ from the start of the run
        return g.toend == 1u && !(g.bits & SPL_B_ATEND);                 // the last one is left for what follows
    }
    const bool prev_space = spl_is_space20<WITH_B>(b, meta, i - 1);      // it starts the chunk (" ?" prefix)
    if (kind == SC_N || kind == SC_O) return before == 0u && !prev_space;
    // letters
    if (before == 0u) {
        if (prev_space) return false;
        const uint64_t p = spl_char_start(b, i - 1);
        if (b(p) == 0x27u && spl_single_oish_start<WITH_B>(b, meta, n, p, i) && spl_contraction_len_gpt2(b, n, i) != 0u) return false;
        return true;
    }
    if (before <= 2u) {   // second or third letter of a run that follows a contraction apostrophe
        uint64_t s = i;
        for (uint32_t c = 0; c < before; ++c) s = spl_char_start(b, s - 1);
        if (s >= 1 && b(s - 1) == 0x27u && spl_single_oish_start<WITH_B>(b, meta, n, s - 1, s)) {
            const uint32_t clen = spl_contraction_len_gpt2(b, n, s);
            return clen != 0u && before == clen - 1u;
        }
    }
    return false;
}
