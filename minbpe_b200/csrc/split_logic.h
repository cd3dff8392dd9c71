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

// ---- the o200k pattern (GPT-4o, tiktoken o200k_base) on scans of its own --------------------------------------------
//   [^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+(?i:'s|'t|'re|'ve|'m|'ll|'d)?
//  |[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*(?i:'s|'t|'re|'ve|'m|'ll|'d)?
//  |\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n/]*|\s*[\r\n]+|\s+(?!\S)|\s+
// Derivation: DESIGN.md §17.  Words are runs of "case letters" (Lu/Lt, Ll, Lm/Lo and the marks \p{M}, which are no \p{L});
// a run is cut at an upper-case letter whose last non-Lm/Lo/M letter in front is lower-case, and at the upper-case tail of a
// run that has no lower-case letter or Lm/Lo/M after it.  What a character does at the edge of a run depends on how far the
// matches before it reach (a mark is eaten by " ?[^\s\p{L}\p{N}]+", a '/' or newline by its tail "[\r\n/]*", an apostrophe
// by a contraction), which no run length bounds.  So the forward scan is a small automaton: its value is the map
// state-before -> state-after of a stretch of text, and maps compose.  The backward scan is SplBwd's over the o200k runs,
// plus "every letter from here to the end of the word is upper-case".
//
// meta bits 5-7: the case class of the character, from the o200k class table (bpe_o200k_table); 0 = not a case letter
#define SM_CASE_SHIFT 5u
#define SM_CASE (7u << SM_CASE_SHIFT)
#define SC_CU 1u   // \p{Lu} \p{Lt}: upper-case only
#define SC_CL 2u   // \p{Ll}: lower-case only
#define SC_CB 3u   // \p{Lm} \p{Lo}: both classes
#define SC_CM 4u   // \p{M}: both classes, and not \p{L}
SPL_HD uint32_t spl_case(uint32_t m) { return (m & SM_CASE) >> SM_CASE_SHIFT; }
// run kind under o200k: case letters (marks included) form one kind; digits, whitespace and the rest as spl_kind
#define SPL_KIND_WORD 8u
SPL_HD uint32_t spl_kind_o200k(uint32_t m) { return spl_case(m) ? SPL_KIND_WORD : spl_kind(m & SM_CLS); }

// automaton states: what the match that holds a character does with the next one
#define SO_X 0u    // nothing carries over: the next character starts from scratch (also: an O character taken as the
                   // [^\r\n\p{L}\p{N}] prefix of the word that follows, the last letter of a contraction)
#define SO_OM 1u   // inside " ?[^\s\p{L}\p{N}]+": takes further O characters and marks
#define SO_TL 2u   // inside its tail [\r\n/]*
#define SO_WN 3u   // inside a word; no Lu/Lt/Ll letter yet (only Lm/Lo/M)
#define SO_WU 4u   // inside a word; the last letter that is not Lm/Lo/M is upper-case
#define SO_WL 5u   // inside a word; ... lower-case
#define SO_C1 6u   // inside a contraction, one letter to go
#define SO_C2 7u   // ... two letters to go
#define SO_D1 8u   // inside \p{N}{1,3}, one digit taken
#define SO_D2 9u   // ... two digits taken
#define SO_NSTATES 10u
SPL_HD bool spl_o_in_word(uint32_t t) { return t == SO_WN || t == SO_WU || t == SO_WL; }

// forward value: 4 bits per state s = the state after the stretch when entered in state s
struct SplFwdO {
    uint64_t map;
};
SPL_HD SplFwdO spl_fwdo_identity() {
    SplFwdO r; r.map = 0;
    for (uint32_t s = 0; s < SO_NSTATES; ++s) r.map |= (uint64_t)s << (4 * s);
    return r;
}
SPL_HD SplFwdO spl_fwdo_const(uint32_t to) {
    SplFwdO r; r.map = 0;
    for (uint32_t s = 0; s < SO_NSTATES; ++s) r.map |= (uint64_t)to << (4 * s);
    return r;
}
SPL_HD void spl_fwdo_set(SplFwdO &f, uint32_t s, uint32_t to) { f.map = (f.map & ~(0xfull << (4 * s))) | ((uint64_t)to << (4 * s)); }
// the state after the stretch when the text before it left state s (the text starts in SO_X)
SPL_HD uint32_t spl_fwdo_state(SplFwdO f, uint32_t s = SO_X) { return (uint32_t)(f.map >> (4 * s)) & 0xfu; }
// a = everything to the left, b = what follows it
SPL_HD SplFwdO spl_fwdo_combine(SplFwdO a, SplFwdO b) {
    SplFwdO r; r.map = 0;
    for (uint32_t s = 0; s < SO_NSTATES; ++s) r.map |= (uint64_t)spl_fwdo_state(b, spl_fwdo_state(a, s)) << (4 * s);
    return r;
}

// first byte of the character after the one that starts at byte j (n if none)
template <class Meta>
SPL_HD uint64_t spl_next_char(const Meta &meta, uint64_t n, uint64_t j) {
    uint64_t k = j + 1;
    while (k < n && k < j + 4 && !(meta(k) & SM_START)) ++k;
    return k < n ? k : n;
}
// contraction after the apostrophe, with its letters inside the same text (WITH_B: no boundary byte among them)
template <bool WITH_B, class Bytes, class Meta>
SPL_HD uint32_t spl_contraction_len_o200k(const Bytes &b, const Meta &meta, uint64_t n, const uint8_t *contr, uint64_t s) {
    if (s >= n || (WITH_B && (meta(s) & SM_CLS) == SC_B)) return 0;
    const uint32_t clen = spl_contraction_len(b, n, contr, s);
    if (WITH_B && clen == 3u && (meta(spl_next_char(meta, n, s)) & SM_CLS) == SC_B) return 0;
    return clen;
}

// element of byte j: the transition of the character that starts there (identity on its other bytes)
template <bool WITH_B, class Bytes, class Meta>
SPL_HD SplFwdO spl_fwdo_elem(uint64_t j, uint64_t n, const Bytes &b, const Meta &meta, const uint8_t *contr) {
    const uint32_t m = meta(j);
    if (!(m & SM_START)) return spl_fwdo_identity();
    const uint32_t cls = m & SM_CLS, cs = spl_case(m);
    if (WITH_B && cls == SC_B) return spl_fwdo_const(SO_X);        // the next text starts from scratch
    if (cls == SC_SP) return spl_fwdo_const(SO_X);
    SplFwdO f;
    if (cls == SC_N) {
        f = spl_fwdo_const(SO_D1);
        spl_fwdo_set(f, SO_D1, SO_D2); spl_fwdo_set(f, SO_D2, SO_X);
    } else if (cls == SC_NL) {                                       // the tail of an O match takes newlines
        f = spl_fwdo_const(SO_X);
        spl_fwdo_set(f, SO_OM, SO_TL); spl_fwdo_set(f, SO_TL, SO_TL);
    } else if (cs != 0u) {                                           // case letter or mark
        const uint32_t fresh = cs == SC_CU ? SO_WU : cs == SC_CL ? SO_WL : SO_WN;
        f = spl_fwdo_const(fresh);
        if (cs == SC_CM) spl_fwdo_set(f, SO_OM, SO_OM);              // a mark is also [^\s\p{L}\p{N}]
        spl_fwdo_set(f, SO_C2, SO_C1); spl_fwdo_set(f, SO_C1, SO_X);
        if (cs == SC_CB || cs == SC_CM) { spl_fwdo_set(f, SO_WU, SO_WU); spl_fwdo_set(f, SO_WL, SO_WL); }   // SO_WN stays
    } else {                                                         // O, apostrophe, '/'
        const uint64_t jn = spl_next_char(meta, n, j);
        const uint32_t start = (jn < n && spl_case(meta(jn)) != 0u) ? SO_X : SO_OM;   // starts a match: word prefix or O match
        const uint32_t clen = cls == SC_AP ? spl_contraction_len_o200k<WITH_B>(b, meta, n, contr, jn) : 0u;
        const uint32_t after_word = clen == 3u ? SO_C2 : clen == 2u ? SO_C1 : start;
        f = spl_fwdo_const(j > 0 && spl_is_space20<WITH_B>(b, meta, j - 1) ? SO_OM : start);   // " ?[^\s\p{L}\p{N}]+" from the space
        spl_fwdo_set(f, SO_OM, SO_OM);
        spl_fwdo_set(f, SO_TL, b(j) == 0x2Fu ? SO_TL : start);
        spl_fwdo_set(f, SO_WN, after_word); spl_fwdo_set(f, SO_WU, after_word); spl_fwdo_set(f, SO_WL, after_word);
    }
    return f;
}

// backward value: SplBwd over the o200k runs, plus allu = every character of the run from this byte on is Lu/Lt
struct SplBwdO {
    uint32_t toend;
    uint32_t bits;   // nlah | atend << 1 | last << 2 | allu << 3
};
#define SPL_B_ALLU 8u
SPL_HD SplBwdO spl_bwdo_identity() { SplBwdO r; r.toend = 0; r.bits = SPL_B_ALLU; return r; }
// a = what comes first in the text, b = everything to the right of it
SPL_HD SplBwdO spl_bwdo_combine(SplBwdO a, SplBwdO b) {
    if (a.bits & SPL_B_LAST) return a;
    SplBwdO r;
    r.toend = a.toend + b.toend;
    r.bits = (b.bits & (SPL_B_ATEND | SPL_B_LAST)) | ((a.bits | b.bits) & SPL_B_NLAH) | (a.bits & b.bits & SPL_B_ALLU);
    return r;
}
template <bool WITH_B = false>
SPL_HD SplBwdO spl_bwdo_elem(uint64_t i, uint64_t n, uint32_t m, uint32_t mnext) {
    const uint32_t cls = m & SM_CLS;
    const bool last = (i + 1 == n) || spl_kind_o200k(mnext) != spl_kind_o200k(m);
    const bool text_ends = (i + 1 == n) || (WITH_B && (mnext & SM_CLS) == SC_B);
    SplBwdO r;
    r.toend = (m & SM_START) ? 1u : 0u;
    r.bits = (cls == SC_NL ? SPL_B_NLAH : 0u) | (spl_case(m) == SC_CU ? SPL_B_ALLU : 0u);
    if (last) r.bits |= SPL_B_LAST | (text_ends ? SPL_B_ATEND : 0u);
    return r;
}

// Does a chunk start at byte i (the first byte of a character)?  t = the automaton state before i (spl_fwdo_state of the
// inclusive forward value at byte i-1; anything for i == 0), g = inclusive backward value at byte i.  Reads b() and meta()
// at most 1 byte before and 9 bytes after i.  WITH_B as for spl_chunk_start.
template <bool WITH_B = false, class Bytes, class Meta>
SPL_HD bool spl_chunk_start_o200k(uint64_t i, uint64_t n, uint32_t t, SplBwdO g, const Bytes &b, const Meta &meta,
                                  const uint8_t *contr) {
    if (i == 0) return true;
    const uint32_t m = meta(i), cls = m & SM_CLS, cs = spl_case(m);
    if (WITH_B && cls == SC_B) return false;
    const uint32_t mp = meta(i - 1), pcls = mp & SM_CLS, pcs = spl_case(mp);   // every byte of a character has its meta
    if (cls == SC_N) return t != SO_D1 && t != SO_D2;                // \p{N}{1,3}
    if (cls == SC_SP || cls == SC_NL) {                              // as spl_chunk_start, with "the tail takes newlines" from t
        const bool is_nl = cls == SC_NL;
        const bool in_run = pcls == SC_SP || pcls == SC_NL;
        const bool is_w2s = (t == SO_OM || t == SO_TL) ? !is_nl : !in_run;
        const bool nlah = (g.bits & SPL_B_NLAH) != 0, atend = (g.bits & SPL_B_ATEND) != 0;
        const bool is_w3s = !nlah && ((pcls == SC_NL && t != SO_TL) || is_w2s);
        return (is_w2s && nlah) || (is_w3s && (atend || g.toend >= 2u)) || (g.toend == 1u && !atend && !is_nl);
    }
    if (cs == 0u) {                                                  // O, apostrophe, '/'
        if (t == SO_OM) return false;
        if (t == SO_TL) return b(i) != 0x2Fu;
        if (spl_o_in_word(t)) return !(cls == SC_AP && spl_contraction_len_o200k<WITH_B>(b, meta, n, contr, i + 1) != 0u);
        return !spl_is_space20<WITH_B>(b, meta, i - 1);
    }
    // case letters and marks
    if (t == SO_OM) return cs != SC_CM;
    if (t == SO_C1 || t == SO_C2) return false;
    if (t == SO_TL) return true;
    if (spl_o_in_word(t))                                            // a case boundary inside the word
        return cs == SC_CU && (t == SO_WL || ((pcs == SC_CB || pcs == SC_CM) && (g.bits & SPL_B_ALLU)));
    return !(pcls == SC_SP || (pcs == 0u && (pcls == SC_O || pcls == SC_AP)));   // a [^\r\n\p{L}\p{N}] prefix starts it
}
