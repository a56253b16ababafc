// tests/shim/nvbowtie_mapping_b200.cu -- the translation unit that REPLACES nvBowtie/bowtie2/cuda/mapping.cu in a build of nvBowtie
// against libnvbio_b200.so: the same entry points (map, map_exact, map_approx, map_whole_read, gather_ranges; mapping.h), defined by
// include/nvbio_b200/shim/nvbowtie_mapping.h.
#define NVBIO_B200_DEFINE_NVBOWTIE_MAPPING
#include <nvbio_b200/shim/nvbowtie_mapping.h>

// the shim's call counters, for the harness (which declares this weak: the build linked against nvBowtie's mapping.cu has none)
extern "C" void nvbowtie_shim_calls(unsigned long long* mapped, unsigned long long* fallbacks)
{
    *mapped = nvbio::b200::stats().fm_rank; *fallbacks = nvbio::b200::stats().fallbacks;
}
