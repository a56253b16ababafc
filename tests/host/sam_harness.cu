// tests/host/sam_harness.cu -- TEST INFRASTRUCTURE.
// Runs the per-record routines of nvb_sam_format (sam_core.cuh) serially on the CPU: sam_line_size per record, the exclusive scan of the
// sizes and the rejection tally, and sam_compose of every line that fits `capacity`, its 32 lanes one after another.  All pointers are
// HOST pointers.  Built by tests/test_sam_host.py.
#include "../../nvbio_b200/csrc/sam_core.cuh"

using namespace nvb;

extern "C" void hh_sam(const uint8_t* records, const uint64_t* in_off, uint32_t n, const char* ref_names, const uint32_t* ref_off,
                       uint32_t n_refs, char* text, uint64_t capacity, uint64_t* offsets, uint32_t* rejected)
{
    uint64_t* sizes = new uint64_t[(size_t)n + 1];
    rejected[0] = 0u; rejected[1] = 0xFFFFFFFFu;
    for (uint32_t i = 0; i < n; ++i) {
        const uint64_t b = in_off[i], e = in_off[i + 1];
        sizes[i] = e >= b ? sam_line_size(records + b, e - b, n_refs, ref_off) : 0u;
        if (!sizes[i]) { ++rejected[0]; if (rejected[1] == 0xFFFFFFFFu) rejected[1] = i; }
    }
    offsets[0] = 0u;
    for (uint32_t i = 0; i < n; ++i) offsets[i + 1] = offsets[i] + sizes[i];
    for (uint32_t i = 0; i < n && offsets[i + 1] <= capacity; ++i)
        if (sizes[i])
            for (uint32_t lane = 0; lane < 32u; ++lane) sam_compose(records + in_off[i], sizes[i], ref_names, ref_off, text + offsets[i], lane, 32u);
    delete[] sizes;
}
