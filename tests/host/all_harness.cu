// tests/host/all_harness.cu -- TEST INFRASTRUCTURE.
// The selection rule of nvb_seed_extend_all run serially on the CPU with the routines the kernels use (reportable, make_best_key,
// end_strand, select_distinct in pipeline_core.cuh): pair_cand_scatter_kernel's filter, the segmented sort's order and
// all_select_kernel's walk over one read's candidates.  Built by tests/test_all_host.py.
#include "../../nvbio_b200/csrc/pipeline_core.cuh"
#include <algorithm>
#include <vector>

using namespace nvb;

// one read's n candidates (score, tie index, end, strand, sink.x); writes the admitted candidates' indices in rank order, returns their number
extern "C" uint32_t hh_select_all(uint32_t n, const int32_t* score, const uint32_t* tie, const uint32_t* end, const uint8_t* strand,
                                  const uint32_t* sink_x, uint32_t len, int32_t min_score, uint32_t k, uint32_t* out)
{
    std::vector<uint32_t> idx;
    for (uint32_t i = 0; i < n; ++i)
        if (reportable(score[i], make_uint2(sink_x[i], 0u), min_score)) idx.push_back(i);
    std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return make_best_key(score[a], tie[a]) > make_best_key(score[b], tie[b]); });
    std::vector<unsigned long long> es(idx.size());
    for (size_t i = 0; i < idx.size(); ++i) es[i] = end_strand(end[idx[i]], strand[idx[i]]);
    const uint32_t m = select_distinct(es.data(), idx.data(), (uint32_t)idx.size(), len, k);
    for (uint32_t i = 0; i < m; ++i) out[i] = idx[i];
    return m;
}
