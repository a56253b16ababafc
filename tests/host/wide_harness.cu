// tests/host/wide_harness.cu -- TEST INFRASTRUCTURE.
// The wide (32-byte) k-mer table on the host: a mirror of nvb_fm_build_ktab_wide's fill pass (the level passes are those of
// hh_fm_build_ktab), and fm_match_locate_one / fm_match_one over an index at any table level (nvb_fm_index.ktab_located 2..5), so
// that the wide table can be checked against the 16-byte one seed by seed.  The rows helpers come with rows_harness.cu.
#include "rows_harness.cu"

static FmIndex mk_level(const uint32_t* bwt_occ, const uint32_t* full_sa, const uint32_t* L2, uint32_t n, uint32_t primary,
                        const uint32_t* ktab, uint32_t ktab_k, uint32_t level, const uint32_t* rows) {
    nvb_fm_index c; c.d_bwt_occ = bwt_occ; c.d_ssa = full_sa; c.length = n; c.primary = primary;
    for (int i = 0; i < 5; ++i) c.L2[i] = L2[i];
    c.sa_interval = 1; c.d_ktab = (const nvb_uint2*)ktab; c.ktab_k = ktab_k; c.ktab_located = level;
    c.d_rows = (const nvb_uint2*)rows;
    if (!valid_fmindex(&c)) abort();
    return make_fmindex(&c);
}

extern "C" {

// 8-byte entries {x, y} (hh_fm_build_ktab) -> 32-byte entries, as fm_ktab32_fill_kernel writes them
void hw_build_wide(const uint32_t* ktab8, const uint32_t* full_sa, const uint32_t* text_words, uint32_t n, uint32_t k, uint32_t* ktab32) {
    for (uint64_t v = 0; v < (1ull << (2u * k)); ++v) {
        uint32_t w[8];
        ktab_wide_fill(full_sa, text_words, n, ktab8[2 * v], ktab8[2 * v + 1], w);
        for (int i = 0; i < 8; ++i) ktab32[8 * v + i] = w[i];
    }
}

// out[3i..3i+2] = (status, x, y) of every query over the table at `level` (rows is used at levels 3 and 5); split = 0: one FM_WHOLE
// call, 1: FM_DEFER then FM_RESUME for what it hands back.  Returns the number of queries handed back (split) or 0.
uint32_t hw_match_locate(const uint32_t* bwt_occ, const uint32_t* full_sa, const uint32_t* L2, uint32_t n, uint32_t primary,
                         const uint32_t* genome, const uint32_t* words, uint32_t bits, const uint32_t* off, const uint32_t* len, uint32_t nq,
                         const uint32_t* ktab, uint32_t ktab_k, uint32_t level, const uint32_t* rows, int split, uint32_t* out) {
    const FmIndex f = mk_level(bwt_occ, full_sa, L2, n, primary, ktab, ktab_k, level, rows);
    uint32_t deferred = 0;
    for (uint32_t i = 0; i < nq; ++i) {
        uint32_t x = 0, y = 0, st = 0;
        if (!split) {
            st = bits == 2 ? fm_match_locate_one<2, true>(f, genome, words, off[i], len[i], x, y)
                           : fm_match_locate_one<4, true>(f, genome, words, off[i], len[i], x, y);
        } else {
            st = bits == 2 ? fm_match_locate_one<2, true, FM_DEFER>(f, genome, words, off[i], len[i], x, y)
                           : fm_match_locate_one<4, true, FM_DEFER>(f, genome, words, off[i], len[i], x, y);
            if (st == FM_DEFERRED) {
                ++deferred;
                st = bits == 2 ? fm_match_locate_one<2, true, FM_RESUME>(f, genome, words, off[i], len[i], x, y)
                               : fm_match_locate_one<4, true, FM_RESUME>(f, genome, words, off[i], len[i], x, y);
            }
        }
        if (st == FM_EMPTY) x = y = 0;                       // (x, y) are only defined for the other two states
        out[3 * i] = st; out[3 * i + 1] = x; out[3 * i + 2] = y;
    }
    return deferred;
}

// fm_match_one (ranges) over the table at `level`, match flags as nvb_fm_match takes them
void hw_match(const uint32_t* bwt_occ, const uint32_t* full_sa, const uint32_t* L2, uint32_t n, uint32_t primary,
              const uint32_t* words, uint32_t bits, const uint32_t* off, const uint32_t* len, uint32_t nq, uint32_t flags,
              const uint32_t* ktab, uint32_t ktab_k, uint32_t level, uint32_t* out_xy) {
    const FmIndex f = mk_level(bwt_occ, full_sa, L2, n, primary, ktab, ktab_k, level, nullptr);
    for (uint32_t i = 0; i < nq; ++i) {
        uint32_t x, y;
        if (bits == 2) fm_match_one<2, true>(f, words, off[i], len[i], flags, x, y);
        else           fm_match_one<4, true>(f, words, off[i], len[i], flags, x, y);
        out_xy[2 * i] = x; out_xy[2 * i + 1] = y;
    }
}

} // extern "C"
