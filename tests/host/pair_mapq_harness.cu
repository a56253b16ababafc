// tests/host/pair_mapq_harness.cu -- TEST INFRASTRUCTURE.
// Runs the pair rule of nvb_seed_extend_paired_mapq (PairSecond / pair_combinations in pipeline_core.cuh) and its paired MAPQ serially on
// the CPU, as pair_second_kernel calls them, so that both can be checked without a GPU: the MAPQ against nvBowtie's own BowtieMapq2 on
// paired alignments (tests/golden/mapq_paired.npz), the rule against a Python restatement.  Built by tests/test_pair_mapq.py.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"

using namespace nvb;

// the paired MAPQ of pair_second_kernel for mate scores (s1, s2) and a second pair (t1 + t2) when kind == 1
extern "C" void hh_bowtie_mapq2_paired(const int32_t* s1, const int32_t* s2, const uint8_t* kind, const int32_t* t1, const int32_t* t2,
                                       const uint32_t* len1, const uint32_t* len2, const int32_t* match_bonus, const int32_t* min1,
                                       const int32_t* min2, uint32_t n, uint8_t* mapq)
{
    for (uint32_t i = 0; i < n; ++i)
        mapq[i] = (uint8_t)bowtie_mapq2(s1[i] + s2[i], kind[i] == 1, t1[i] + t2[i], (int32_t)(len1[i] + len2[i]) * match_bonus[i],
                                        min1[i] + min2[i], match_bonus[i] == 0);
}

// the second-best pair of n pairs.  Mate m of pair p (index i = m * n + p): merged, sorted candidates end/score/tie[seg[i], seg[i] + cnt[i])
// with the forward ones first (n_fw[i]), read length len[i], P*'s mate (star_end[i], star_strand[i]).  Rescue k of pair p (k < n_resc[p]):
// anchor r_anchor[2p + k], pair score r_score, anchor end / strand / tie r_aend / r_astrand / r_atie, rescued end r_oend.
extern "C" void hh_pair_second(uint32_t n, const uint32_t* seg, const uint32_t* n_fw, const uint32_t* cnt, const uint32_t* len,
                               const uint32_t* end, const int32_t* score, const uint32_t* tie,
                               const uint32_t* star_end, const uint32_t* star_strand, uint32_t min_frag, uint32_t max_frag,
                               const uint32_t* n_resc, const uint32_t* r_anchor, const int32_t* r_score, const uint32_t* r_aend,
                               const uint32_t* r_astrand, const uint32_t* r_atie, const uint32_t* r_oend,
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
        pair_combinations(m, min_frag, max_frag, ps);
        for (uint32_t k = 0; k < n_resc[p]; ++k) {
            const uint32_t j = 2u * p + k;
            ps.offer_rescue((int)r_anchor[j], r_score[j], r_aend[j], r_astrand[j], r_atie[j], r_oend[j]);
        }
        has[p] = ps.has ? 1 : 0; out_score[p] = ps.score;
        for (int k = 0; k < 2; ++k) { out_end[k * n + p] = ps.end[k]; out_strand[k * n + p] = ps.strand[k]; }
    }
}
