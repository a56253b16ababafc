// tests/host/pair_policy_harness.cu -- TEST INFRASTRUCTURE.
// Runs the paired-end policy rules of pipeline_core.cuh (pe_frame, pe_concordant, pe_rescue_window and the general pair_combinations)
// serially on the CPU, as pair_classify_kernel, pair_finalize_kernel and pair_second_kernel call them, so that they can be checked
// without a GPU: the framing against nvBowtie's own frame_opposite_mate, the rest against Python restatements.  Built by
// tests/test_pair_policy.py.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"

using namespace nvb;

// pe_frame(policy[i], a[i], t[i]) -> (left[i], strand[i]); policy in NVB_PE_* numbering
extern "C" void hp_frame(const uint32_t* policy, const uint32_t* a, const uint32_t* t, uint32_t n, uint8_t* left, uint8_t* strand)
{
    for (uint32_t i = 0; i < n; ++i) { const PeFrame f = pe_frame(policy[i], a[i], t[i]); left[i] = f.left ? 1 : 0; strand[i] = (uint8_t)f.strand; }
}

// pe_concordant of mate 1 (t1, b1, e1) and mate 2 (t2, b2, e2) under one policy / flags / fragment range
extern "C" void hp_concordant(uint32_t policy, uint32_t flags, uint32_t min_frag, uint32_t max_frag, const uint32_t* t1, const uint32_t* b1,
                              const uint32_t* e1, const uint32_t* t2, const uint32_t* b2, const uint32_t* e2, uint32_t n, uint8_t* out)
{
    for (uint32_t i = 0; i < n; ++i) out[i] = pe_concordant(policy, flags, t1[i], b1[i], e1[i], t2[i], b2[i], e2[i], min_frag, max_frag) ? 1 : 0;
}

// pe_rescue_window of anchor a[i] on strand t[i] at [b[i], e[i]) -> (window begin, window length, strand of the other mate)
extern "C" void hp_rescue_window(uint32_t policy, uint32_t flags, uint32_t max_frag, uint32_t genome_len, const uint32_t* a, const uint32_t* t,
                                 const uint32_t* b, const uint32_t* e, uint32_t n, uint32_t* wb, uint32_t* wl, uint32_t* strand)
{
    for (uint32_t i = 0; i < n; ++i) strand[i] = pe_rescue_window(policy, flags, a[i], t[i], b[i], e[i], max_frag, genome_len, wb[i], wl[i]);
}

// the second-best pair of n pairs from the concordant combinations alone (pair_combinations under policy / flags; layout as
// pair_mapq_harness.cu's hh_pair_second)
extern "C" void hp_pair_combinations(uint32_t n, uint32_t policy, uint32_t flags, const uint32_t* seg, const uint32_t* n_fw, const uint32_t* cnt,
                                     const uint32_t* len, const uint32_t* end, const int32_t* score, const uint32_t* tie,
                                     const uint32_t* star_end, const uint32_t* star_strand, uint32_t min_frag, uint32_t max_frag,
                                     uint8_t* has, int32_t* out_score, uint32_t* out_end, uint32_t* out_strand)
{
    for (uint32_t p = 0; p < n; ++p) {
        PairSecond ps;
        ps.init(star_end[p], star_strand[p], len[p], star_end[n + p], star_strand[n + p], len[n + p]);
        MateCands m[2];
        for (int k = 0; k < 2; ++k) {
            const uint32_t i = k * n + p;
            m[k].end = end + seg[i]; m[k].score = score + seg[i]; m[k].tie = tie + seg[i]; m[k].n_fw = n_fw[i]; m[k].n = cnt[i]; m[k].len = len[i];
        }
        pair_combinations(m, policy, flags, min_frag, max_frag, ps);
        has[p] = ps.has ? 1 : 0; out_score[p] = ps.score;
        for (int k = 0; k < 2; ++k) { out_end[k * n + p] = ps.end[k]; out_strand[k * n + p] = ps.strand[k]; }
    }
}
