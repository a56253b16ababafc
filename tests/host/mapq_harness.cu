// tests/host/mapq_harness.cu -- TEST INFRASTRUCTURE.
// Runs bowtie_mapq2 (pipeline_core.cuh, the MAPQ of nvb_seed_extend_mapq) serially on the CPU, as pipe_mapq_kernel calls it, so that the
// host build can be checked against nvBowtie's own BowtieMapq2 (tests/golden/mapq.npz) without a GPU.  Built by tests/test_mapq.py.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"

using namespace nvb;

extern "C" void hh_bowtie_mapq2(const int32_t* best, const uint8_t* has_second, const int32_t* second, const uint32_t* len,
                                const int32_t* match_bonus, const int32_t* min_score, uint32_t n, uint8_t* mapq)
{
    for (uint32_t i = 0; i < n; ++i)
        mapq[i] = (uint8_t)bowtie_mapq2(best[i], has_second[i] != 0, second[i], (int32_t)len[i] * match_bonus[i], min_score[i], match_bonus[i] == 0);
}
