// tests/host/bam_all_harness.cu -- TEST INFRASTRUCTURE.
// Runs nvb_bam_records_all's per-read planning (bam_plan_read_all, bam_core.cuh) serially on the CPU: the count pass, the scan of the
// record counts, the plan pass, the scan of the sizes, and bam_compose of every record, its 32 lanes one after another.  The nvb_bam_all_in
// it takes holds HOST pointers.  Built by tests/test_all_host.py.
#include "../../nvbio_b200/csrc/bam_core.cuh"
#include <vector>

using namespace nvb;

// records must hold the whole output; offsets [n_reads + capacity + 1]; returns the number of records
extern "C" uint32_t hh_bam_all(const nvb_bam_all_in* in, uint32_t n_reads, uint8_t* records, uint64_t* offsets, uint32_t* counts)
{
    const nvb_bam_in& I = in->base;
    const nvb_finish_out& F = I.finish;
    const uint32_t slots = n_reads + in->capacity;
    std::vector<uint4> rec(slots + 1);
    std::vector<uint32_t> cores(8 * (size_t)slots + 8), rec_first(n_reads + 1);
    std::vector<uint64_t> sizes(slots + 1, 0u);
    BamIn b;
    b.reads = make_strset(&I.reads); b.quals = I.d_read_quals;
    b.n_ops = I.d_n_ops; b.begin = (const uint2*)I.d_begin; b.strand = I.d_strand;
    b.cigar = F.d_cigar; b.max_cigar = F.max_cigar; b.n_cigar = F.d_n_cigar;
    b.md = F.d_md; b.max_md = F.max_md; b.md_len = F.d_md_len; b.edits = F.d_edits;
    b.score = I.d_score; b.mapq = I.d_mapq; b.second = I.d_second_score; b.pair_flags = nullptr;
    b.contig_begin = I.d_contig_begin; b.n_contigs = I.n_contigs;
    b.names = I.d_names; b.name_off = I.d_name_offsets; b.n = slots; b.rec = rec.data();
    uint32_t cnt[3] = { 0u, 0u, 0u };
    rec_first[0] = 0u;
    for (uint32_t r = 0; r < n_reads; ++r)
        rec_first[r + 1] = rec_first[r] + bam_plan_read_all(b, r, in->d_first, in->capacity, nullptr, nullptr, nullptr, nullptr, cnt);
    for (uint32_t r = 0; r < n_reads; ++r)
        bam_plan_read_all(b, r, in->d_first, in->capacity, rec_first.data(), rec.data(), cores.data(), sizes.data(), cnt);
    const uint32_t n = rec_first[n_reads];
    offsets[0] = 0u;
    for (uint32_t k = 0; k < slots; ++k) offsets[k + 1] = offsets[k] + sizes[k];
    counts[0] = n; counts[1] = cnt[0]; counts[2] = cnt[1]; counts[3] = cnt[2];
    for (uint32_t k = 0; k < n; ++k)
        for (uint32_t lane = 0; lane < 32u; ++lane) {
            if (b.reads.bits == 2) bam_compose<2, true>(b, k, cores.data() + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
            else                   bam_compose<4, true>(b, k, cores.data() + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
        }
    return n;
}
