// tests/host/full_tb_harness.cu -- TEST INFRASTRUCTURE.
// Runs the rescued-mate traceback of nvb_seed_extend_paired_traceback serially on the CPU with the shipped routines, so that its window
// cuts can be checked without a GPU: the lanes of gotoh_full_warp_traceback_kernel (FullTbLane, gotoh_full_core.cuh) emulated in lockstep
// over the rows [r0, sink.x) that full_traceback_first_row (pipeline_core.cuh) keeps, the step-major matrix walked by gotoh_full_walk,
// against gotoh_full_impl2 + the row-major walk on the whole window.  Built by tests/test_paired_traceback_host.py.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"
#include "../../nvbio_b200/csrc/gotoh_full_core.cuh"
#include <vector>

using namespace nvb;

// one alignment through the emulated warp: lane l's step t is FullTbLane::row of text row t - l; a lane reads the (H, E, symbol) its left
// neighbour produced at step t - 1, so the lanes are visited right to left within a step
template <int TYPE, int W>
static uint32_t warp_emulation(const GotohScheme& S, const uint8_t* pat, uint32_t poff, uint32_t M, const uint8_t* quals, const uint8_t* txt, uint32_t r0,
                               uint32_t R, uint32_t sink_y, uint8_t* ops, uint32_t max_ops, uint32_t& sx, uint32_t& sy)
{
    constexpr int NW = FullTbLane<W>::NW;
    const int32_t INF = SHRT_MIN - (S.pgo < S.pge ? S.pgo : S.pge);
    const uint32_t L = (M + W - 1) / W, steps = R + L - 1;
    std::vector<uint32_t> dirs((size_t)steps * NW * 32u, 0u);
    std::vector<FullTbLane<W>> lane(32);
    int32_t outH[32] = {0}, outE[32] = {0};
    uint32_t outG[32] = {0};
    for (uint32_t l = 0; l < 32; ++l) lane[l].template init<TYPE>(S, (const uint32_t*)pat, 8u, 0u, poff, M, quals, l * W, INF);
    for (uint32_t t = 0; t < steps; ++t) {
        for (int l = 31; l >= 0; --l) {
            const uint32_t r = t - (uint32_t)l;
            if (r >= R || (uint32_t)l >= L) continue;
            int32_t Hl, E; uint32_t g;
            if (l == 0) { full_first_column<TYPE>(S, r0 + r, INF, Hl, E); g = txt[r0 + r]; }
            else        { Hl = outH[l - 1]; E = outE[l - 1]; g = outG[l - 1]; }
            uint32_t dw[NW];
            lane[l].template row<TYPE>(S, g, Hl, E, dw);
            outH[l] = Hl; outE[l] = E; outG[l] = g;
            for (int w = 0; w < NW; ++w) dirs[((size_t)t * NW + w) * 32u + l] = dw[w];
        }
    }
    SinkResult s; s.score = 0; s.x = R; s.y = sink_y;
    return gotoh_full_walk<TYPE>(FullDirsStepMajor{dirs.data(), (uint32_t)W, (uint32_t)NW}, s, ops, max_ops, sx, sy);
}

template <int TYPE>
static uint32_t warp_dispatch(const GotohScheme& S, const uint8_t* pat, uint32_t poff, uint32_t M, const uint8_t* quals, const uint8_t* txt, uint32_t r0,
                              uint32_t R, uint32_t sink_y, uint8_t* ops, uint32_t max_ops, uint32_t& sx, uint32_t& sy)
{
#define HH_W(w) case w: return warp_emulation<TYPE, w>(S, pat, poff, M, quals, txt, r0, R, sink_y, ops, max_ops, sx, sy);
    switch ((M + 31) / 32) { HH_W(1) HH_W(2) HH_W(3) HH_W(4) HH_W(5) HH_W(6) HH_W(7) HH_W(8) HH_W(9) HH_W(10) HH_W(11) HH_W(12) HH_W(13)
                             HH_W(14) HH_W(15) default: return warp_emulation<TYPE, 16>(S, pat, poff, M, quals, txt, r0, R, sink_y, ops, max_ops, sx, sy); }
#undef HH_W
}

// n alignments; patterns / texts as one byte per symbol at p_off / t_off; qtab (256 x 2) and quals may be NULL.  Out: the full window's
// score, sink, source, ops (gotoh_full_impl2 + FullDirsRowMajor walk); r0 of the cut; the cut window's source, ops (warp emulation +
// FullDirsStepMajor walk, source shifted back)
template <int TYPE>
static void run(const GotohScheme& S, int32_t s_max, const uint8_t* pat, const uint32_t* p_off, const uint32_t* p_len, const uint8_t* quals,
                const uint8_t* txt, const uint32_t* t_off, const uint32_t* t_len, uint32_t n, uint32_t max_ops,
                int32_t* score, uint32_t* sink, uint32_t* r0_out, uint32_t* src, uint32_t* n_ops, uint8_t* ops,
                uint32_t* src_cut, uint32_t* n_ops_cut, uint8_t* ops_cut)
{
    for (uint32_t a = 0; a < n; ++a) {
        const uint32_t M = p_len[a], N = t_len[a], rw = (M + 31u) / 32u * 4u;
        std::vector<uint32_t> dirs((size_t)N * rw, 0u);
        std::vector<int2> col((size_t)N + 1);
        const SinkResult r = gotoh_full_impl<TYPE, true>(S, (const uint32_t*)pat, 8u, 0u, p_off[a], M,
                                                         (const uint32_t*)txt, 8u, 0u, t_off[a], N, col.data(), 1, dirs.data(), rw, quals);
        score[a] = r.score; sink[2 * a] = r.x; sink[2 * a + 1] = r.y;
        uint32_t sx = 0, sy = 0;
        n_ops[a] = gotoh_full_walk<TYPE>(FullDirsRowMajor{dirs.data(), rw}, r, ops + (size_t)a * max_ops, max_ops, sx, sy);
        src[2 * a] = sx; src[2 * a + 1] = sy;
        const uint32_t r0 = full_traceback_first_row(TYPE, r.x, r.y, r.score, s_max, S.pgo, S.pge);
        r0_out[a] = r0;
        n_ops_cut[a] = warp_dispatch<TYPE>(S, pat, p_off[a], M, quals, txt + t_off[a], r0, r.x - r0, r.y,
                                           ops_cut + (size_t)a * max_ops, max_ops, sx, sy);
        src_cut[2 * a] = r0 + sx; src_cut[2 * a + 1] = sy;
    }
}

extern "C" void hh_full_tb(int type, int32_t match, int32_t mismatch, int32_t pgo, int32_t pge, int32_t tgo, int32_t tge, const int32_t* qtab,
                           const uint8_t* pat, const uint32_t* p_off, const uint32_t* p_len, const uint8_t* quals,
                           const uint8_t* txt, const uint32_t* t_off, const uint32_t* t_len, uint32_t n, uint32_t max_ops,
                           int32_t* score, uint32_t* sink, uint32_t* r0, uint32_t* src, uint32_t* n_ops, uint8_t* ops,
                           uint32_t* src_cut, uint32_t* n_ops_cut, uint8_t* ops_cut)
{
    nvb_gotoh_scheme sc = {};
    sc.match = match; sc.mismatch = mismatch; sc.pattern_gap_open = pgo; sc.pattern_gap_ext = pge; sc.text_gap_open = tgo; sc.text_gap_ext = tge;
    sc.d_qual_table = qtab;
    const GotohScheme S = make_scheme(&sc);
    int32_t s_max = match > mismatch ? match : mismatch;                 // as the kernel derives it
    if (qtab) { s_max = INT_MIN; for (int i = 0; i < 512; ++i) s_max = qtab[i] > s_max ? qtab[i] : s_max; }
    if (type == NVB_LOCAL)       run<NVB_LOCAL>(S, s_max, pat, p_off, p_len, quals, txt, t_off, t_len, n, max_ops, score, sink, r0, src, n_ops, ops, src_cut, n_ops_cut, ops_cut);
    else if (type == NVB_GLOBAL) run<NVB_GLOBAL>(S, s_max, pat, p_off, p_len, quals, txt, t_off, t_len, n, max_ops, score, sink, r0, src, n_ops, ops, src_cut, n_ops_cut, ops_cut);
    else                         run<NVB_SEMI_GLOBAL>(S, s_max, pat, p_off, p_len, quals, txt, t_off, t_len, n, max_ops, score, sink, r0, src, n_ops, ops, src_cut, n_ops_cut, ops_cut);
}
