// tests/host/shortcut_harness.cu -- TEST INFRASTRUCTURE.
// gapless_job_shortcut (pipeline_core.cuh), the per-job routine of pipe_perfect_jobs_kernel, run serially on the CPU with its one-gap
// check on or off, so that both rules can be compared with each other and with the oracle's banded DP.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"

using namespace nvb;

extern "C" {

// solved[a] = 1 and (score[a], sink_xy[2a..]) when the routine proves the LOCAL band result of job a
void hs_gapless_job_shortcut(const uint32_t* str_words, const uint32_t* genome_words, const uint32_t* po, const uint32_t* M, const uint32_t* to,
                             const uint32_t* N, uint32_t n, uint32_t band, int32_t match, int32_t mismatch, int32_t max_gap_open, int one_gap,
                             uint8_t* solved, int32_t* score, uint32_t* sink_xy) {
    for (uint32_t a = 0; a < n; ++a) {
        int32_t sc = 0; uint32_t sx = 0, sy = 0;
        solved[a] = gapless_job_shortcut(str_words, genome_words, po[a], M[a], to[a], N[a], band, match, mismatch, max_gap_open, sc, sx, sy,
                                         one_gap != 0) ? 1 : 0;
        score[a] = sc; sink_xy[2 * a] = sx; sink_xy[2 * a + 1] = sy;
    }
}

} // extern "C"
