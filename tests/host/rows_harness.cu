// tests/host/rows_harness.cu -- TEST INFRASTRUCTURE.
// fm_match_locate_one compiled for the host over an index with and without the per-row array (nvb_fm_index.ktab_located 3 / 2), in
// the single-call form and in the two-pass form of the seed-match stage, plus a host mirror of fm_rows_kernel.  The table helpers
// (hh_fm_build_ktab, hh_fm_ktab_locate, hh_fm_ktab_context) come with host_harness.cu.
#include "host_harness.cu"

static FmIndex mk_rows(const uint32_t* bwt_occ, const uint32_t* full_sa, const uint32_t* L2, uint32_t n, uint32_t primary,
                       const uint32_t* ktab_ctx, uint32_t ktab_k, const uint32_t* rows) {
    nvb_fm_index c; c.d_bwt_occ = bwt_occ; c.d_ssa = full_sa; c.length = n; c.primary = primary;
    for (int i = 0; i < 5; ++i) c.L2[i] = L2[i];
    c.sa_interval = 1; c.d_ktab = (const nvb_uint2*)ktab_ctx; c.ktab_k = ktab_k; c.ktab_located = rows ? 3u : 2u;
    c.d_rows = (const nvb_uint2*)rows;
    if (!valid_fmindex(&c)) abort();
    return make_fmindex(&c);
}

extern "C" {

// rows[2r] = SA[r], rows[2r + 1] = the 16 symbols before it (what nvb_fm_build_rows writes), r in [0, n]
void hr_build_rows(const uint32_t* full_sa, const uint32_t* text_words, uint32_t n, uint32_t* rows) {
    for (uint64_t r = 0; r <= n; ++r) { rows[2 * r] = full_sa[r]; rows[2 * r + 1] = hh_text_before(text_words, full_sa[r], 16u); }
}

// out[3i..3i+2] = (status, x, y) of every query; split = 0: one FM_WHOLE call, 1: FM_DEFER then FM_RESUME for what it hands back.
// Returns the number of queries handed back (split) or 0.
uint32_t hr_match_locate(const uint32_t* bwt_occ, const uint32_t* full_sa, const uint32_t* L2, uint32_t n, uint32_t primary,
                         const uint32_t* genome, const uint32_t* words, uint32_t bits, const uint32_t* off, const uint32_t* len, uint32_t nq,
                         const uint32_t* ktab_ctx, uint32_t ktab_k, const uint32_t* rows, int split, uint32_t* out) {
    const FmIndex f = mk_rows(bwt_occ, full_sa, L2, n, primary, ktab_ctx, ktab_k, rows);
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

} // extern "C"
