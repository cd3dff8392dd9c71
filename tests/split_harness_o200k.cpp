// tests/split_harness_o200k.cpp — test infrastructure.  Runs the o200k rule of minbpe_b200/csrc/split_logic.h on the CPU
// with both of its scans evaluated tile by tile as k_split.cuh decomposes them (tile aggregates, exclusive scans of the
// aggregates, in-tile scans seeded with the carries), so tests/test_split_rules_o200k.py can pin it against `regex`.
#include <stdint.h>
#include <vector>

#include "../minbpe_b200/csrc/split_logic.h"

struct ByteAcc {
    const uint8_t *p;
    uint32_t operator()(uint64_t i) const { return p[i]; }
};

// cls_table: the o200k table (GPT-4 class | case class << SM_CASE_SHIFT).  hits[j] = position << 8 | length of a text
// boundary (special-token occurrence or document gap): its bytes get class SC_B, and the flags are fixed up as
// k_special_flags does.
template <bool WITH_B>
static void flags_impl(const uint8_t *bytes, uint64_t n, const uint8_t *cls_table, const uint8_t *contr, uint64_t tile,
                       const uint64_t *hits, uint64_t n_hits, uint8_t *flags) {
    if (n == 0) return;
    if (tile == 0) tile = n;
    const ByteAcc B{bytes};
    std::vector<uint8_t> meta(n);
    for (uint64_t i = 0; i < n; ++i) meta[i] = (uint8_t)spl_meta_of(B, i, n, cls_table);
    for (uint64_t j = 0; j < n_hits; ++j)
        for (uint64_t t = 0; t < (hits[j] & 0xff); ++t) { uint8_t &m = meta[(hits[j] >> 8) + t]; m = (uint8_t)((m & SM_START) | SC_B); }
    const ByteAcc M{meta.data()};
    auto fe = [&](uint64_t i) { return spl_fwdo_elem<WITH_B>(i, n, B, M, contr); };
    auto ge = [&](uint64_t i) { return spl_bwdo_elem<WITH_B>(i, n, meta[i], i + 1 < n ? meta[i + 1] : 0); };
    const uint64_t ntiles = (n + tile - 1) / tile;
    std::vector<SplFwdO> fcar(ntiles);
    std::vector<SplBwdO> gcar(ntiles);
    for (uint64_t t = 0; t < ntiles; ++t) {   // 1. tile aggregates
        const uint64_t lo = t * tile, hi = (lo + tile < n) ? lo + tile : n;
        SplFwdO f = spl_fwdo_identity();
        for (uint64_t i = lo; i < hi; ++i) f = spl_fwdo_combine(f, fe(i));
        SplBwdO g = spl_bwdo_identity();
        for (uint64_t i = hi; i > lo; --i) g = spl_bwdo_combine(ge(i - 1), g);
        fcar[t] = f; gcar[t] = g;
    }
    SplFwdO frun = spl_fwdo_identity();       // 2. exclusive scans of the aggregates
    for (uint64_t t = 0; t < ntiles; ++t) { const SplFwdO x = fcar[t]; fcar[t] = frun; frun = spl_fwdo_combine(frun, x); }
    SplBwdO grun = spl_bwdo_identity();
    for (uint64_t t = ntiles; t > 0; --t) { const SplBwdO x = gcar[t - 1]; gcar[t - 1] = grun; grun = spl_bwdo_combine(x, grun); }
    std::vector<SplBwdO> gv(tile);            // 3. in-tile scans seeded with the carries, then the rule
    for (uint64_t t = 0; t < ntiles; ++t) {
        const uint64_t lo = t * tile, hi = (lo + tile < n) ? lo + tile : n;
        SplBwdO g = gcar[t];
        for (uint64_t i = hi; i > lo; --i) { g = spl_bwdo_combine(ge(i - 1), g); gv[i - 1 - lo] = g; }
        SplFwdO f = fcar[t];
        for (uint64_t i = lo; i < hi; ++i) {
            const uint32_t state = spl_fwdo_state(f);
            flags[i] = (meta[i] & SM_START) && spl_chunk_start_o200k<WITH_B>(i, n, state, gv[i - lo], B, M, contr) ? 1 : 0;
            f = spl_fwdo_combine(f, fe(i));
        }
    }
    for (uint64_t j = 0; j < n_hits; ++j) {
        const uint64_t pos = hits[j] >> 8, len = hits[j] & 0xff;
        flags[pos] = 1;
        for (uint64_t t = 1; t < len; ++t) flags[pos + t] = 0;
        if (pos + len < n) flags[pos + len] = 1;
    }
}

extern "C" int split_logic_flags_o200k(const uint8_t *bytes, uint64_t n, const uint8_t *cls_table, const uint8_t *contr,
                                       uint64_t tile, const uint64_t *hits, uint64_t n_hits, uint8_t *flags) {
    if (n_hits) flags_impl<true>(bytes, n, cls_table, contr, tile, hits, n_hits, flags);
    else flags_impl<false>(bytes, n, cls_table, contr, tile, nullptr, 0, flags);
    return 0;
}
