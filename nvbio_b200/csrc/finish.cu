// finish.cu -- nvb_finish_alignments: the last per-alignment stage before SAM / BAM output (nvBowtie's finish_alignment_kernel,
// nvBowtie/bowtie2/cuda/traceback_inl.h:520-723).  One thread per traced alignment turns (ops, begin, strand) and the read and genome
// beside it into a BAM CIGAR with soft clips, the MD:Z value and NM / XM / XO / XG (finish_alignment, finish_core.cuh).
#include "finish_core.cuh"

namespace nvb {

template <int BITS, bool BE>
__global__ void __launch_bounds__(128)
finish_alignments_kernel(const uint32_t* __restrict__ genome, const uint32_t genome_len, const StrSet reads, const uint32_t n,
                         const uint8_t* __restrict__ ops, const uint32_t max_ops, const uint32_t* __restrict__ n_ops,
                         const uint2* __restrict__ begin, const uint8_t* __restrict__ strand,
                         uint32_t* __restrict__ cigar, const uint32_t max_cigar, uint32_t* __restrict__ n_cigar,
                         char* __restrict__ md, const uint32_t max_md, uint32_t* __restrict__ md_len, uint32_t* __restrict__ edits)
{
    const uint32_t a = blockIdx.x * 128u + threadIdx.x;
    if (a >= n) return;
    const uint2 b = begin[a];
    FinishOut o;
    o.cigar = cigar + (size_t)a * max_cigar; o.max_cigar = max_cigar;
    o.md = md + (size_t)a * max_md; o.max_md = max_md;
    finish_alignment<BITS, BE>(genome, genome_len, reads.words, str_off(reads, a), str_len(reads, a), strand[a],
                               ops + (size_t)a * max_ops, n_ops[a], max_ops, b.x, b.y, o, edits + 4u * (size_t)a);
    n_cigar[a] = o.n_cigar;
    md_len[a] = o.md_len;
}

} // namespace nvb

using namespace nvb;

extern "C" int nvb_finish_alignments(const uint32_t* d_genome, uint32_t genome_len, const nvb_string_set* reads, uint32_t n,
                                     const nvb_best_alignment_out* A, const nvb_finish_out* out, void* stream)
{
    if (!d_genome || !valid_strset(reads) || !A || !out) return NVB_E_INVALID;
    if (!A->d_ops || !A->d_n_ops || !A->d_begin || !A->d_strand || A->max_ops == 0u) return NVB_E_INVALID;
    if (!out->d_cigar || !out->d_n_cigar || !out->d_md || !out->d_md_len || !out->d_edits || out->max_cigar == 0u || out->max_md == 0u)
        return NVB_E_INVALID;
    if (reads->bits == 8) return NVB_E_UNSUPPORTED;
    if (n == 0u) return NVB_OK;
    const StrSet rd = make_strset(reads);
    const cudaStream_t s = as_stream(stream);
    const uint32_t grid = (n + 127u) / 128u;
#define NVB_FINISH_LAUNCH(BITS, BE_)                                                                                                   \
    finish_alignments_kernel<BITS, BE_><<<grid, 128, 0, s>>>(d_genome, genome_len, rd, n, A->d_ops, A->max_ops, A->d_n_ops,          \
                                                            (const uint2*)A->d_begin, A->d_strand, out->d_cigar, out->max_cigar,   \
                                                            out->d_n_cigar, out->d_md, out->max_md, out->d_md_len, out->d_edits)
    if (reads->bits == 2) { if (reads->big_endian) NVB_FINISH_LAUNCH(2, true); else NVB_FINISH_LAUNCH(2, false); }
    else                  { if (reads->big_endian) NVB_FINISH_LAUNCH(4, true); else NVB_FINISH_LAUNCH(4, false); }
#undef NVB_FINISH_LAUNCH
    return (int)cudaGetLastError();
}
