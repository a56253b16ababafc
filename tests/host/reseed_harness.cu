// Host build of nvb_seed_extend_reseed's per-read rules (nvbio_b200/csrc/pipeline_core.cuh) for tests/test_reseed_host.py
#include "../../nvbio_b200/csrc/pipeline_core.cuh"

using namespace nvb;

extern "C" void rh_reseed_offset(const uint32_t* round, const uint32_t* interval, const uint32_t* max_reseed, uint32_t n, uint32_t* out)
{
    for (uint32_t i = 0; i < n; ++i) out[i] = reseed_offset(round[i], interval[i], max_reseed[i]);
}

extern "C" void rh_reseed_read(const uint32_t* range_sum, const uint32_t* range_count, const uint32_t* rep_seeds, const uint8_t* aligned,
                               uint32_t n, uint8_t* out)
{
    for (uint32_t i = 0; i < n; ++i) out[i] = reseed_read(range_sum[i], range_count[i], rep_seeds[i], aligned[i] != 0) ? 1 : 0;
}
