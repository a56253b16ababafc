// tests/host/bam_harness.cu -- TEST INFRASTRUCTURE.
// Runs the per-record routines of nvb_bam_records (bam_core.cuh) serially on the CPU: bam_plan_unit per read / pair, the exclusive scan
// of the sizes, and bam_compose of every record that fits `capacity`, its 32 lanes one after another.  The nvb_bam_in it takes holds HOST
// pointers.  Built by tests/test_bam_host.py.
#include "../../nvbio_b200/csrc/bam_core.cuh"

using namespace nvb;

extern "C" void hh_bam(const nvb_bam_in* in, uint32_t n, uint8_t* records, uint64_t capacity, uint64_t* offsets, uint32_t* counts)
{
    const nvb_finish_out& F = in->finish;
    BamIn b;
    b.reads = make_strset(&in->reads); b.quals = in->d_read_quals;
    b.n_ops = in->d_n_ops; b.begin = (const uint2*)in->d_begin; b.strand = in->d_strand;
    b.cigar = F.d_cigar; b.max_cigar = F.max_cigar; b.n_cigar = F.d_n_cigar;
    b.md = F.d_md; b.max_md = F.max_md; b.md_len = F.d_md_len; b.edits = F.d_edits;
    b.score = in->d_score; b.mapq = in->d_mapq; b.second = in->d_second_score; b.pair_flags = in->d_pair_flags;
    b.contig_begin = in->d_contig_begin; b.n_contigs = in->n_contigs;
    b.names = in->d_names; b.name_off = in->d_name_offsets; b.n = n;
    uint32_t* cores = new uint32_t[8 * (size_t)n + 8];
    uint64_t* sizes = new uint64_t[(size_t)n + 1];
    uint32_t cnt[3] = { 0u, 0u, 0u };
    const uint32_t units = in->d_pair_flags ? n / 2u : n;
    for (uint32_t u = 0; u < units; ++u) bam_plan_unit(b, u, cores, sizes, cnt);
    offsets[0] = 0u;
    for (uint32_t k = 0; k < n; ++k) offsets[k + 1] = offsets[k] + sizes[k];
    counts[0] = n; counts[1] = cnt[0]; counts[2] = cnt[1]; counts[3] = cnt[2];
    for (uint32_t k = 0; k < n && offsets[k + 1] <= capacity; ++k) {
        for (uint32_t lane = 0; lane < 32u; ++lane) {
            if (b.reads.bits == 2) {
                if (b.reads.big_endian) bam_compose<2, true>(b, k, cores + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
                else                    bam_compose<2, false>(b, k, cores + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
            } else {
                if (b.reads.big_endian) bam_compose<4, true>(b, k, cores + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
                else                    bam_compose<4, false>(b, k, cores + 8u * (size_t)k, (uint32_t)sizes[k], records + offsets[k], lane, 32u);
            }
        }
    }
    delete[] cores; delete[] sizes;
}

extern "C" uint32_t hh_reg2bin(int64_t beg, int64_t end) { return bam_reg2bin(beg, end); }
