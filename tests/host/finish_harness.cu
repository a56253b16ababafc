// tests/host/finish_harness.cu -- TEST INFRASTRUCTURE.
// Runs finish_alignment (finish_core.cuh, the per-alignment routine of nvb_finish_alignments) serially on the CPU with the same inputs
// finish_alignments_kernel hands it, so that CIGAR, MD and edit counts can be checked without a GPU.  Built by tests/test_finish_host.py.
#include "../../nvbio_b200/csrc/finish_core.cuh"

using namespace nvb;

template <int BITS, bool BE>
static void run(const uint32_t* genome, uint32_t genome_len, const uint32_t* read_words, const uint32_t* offs, const uint32_t* lens, uint32_t n,
                const uint8_t* strand, const uint8_t* ops, uint32_t max_ops, const uint32_t* n_ops, const uint32_t* begin,
                uint32_t* cigar, uint32_t max_cigar, uint32_t* n_cigar, char* md, uint32_t max_md, uint32_t* md_len, uint32_t* edits)
{
    for (uint32_t a = 0; a < n; ++a) {
        FinishOut o;
        o.cigar = cigar + (size_t)a * max_cigar; o.max_cigar = max_cigar;
        o.md = md + (size_t)a * max_md; o.max_md = max_md;
        finish_alignment<BITS, BE>(genome, genome_len, read_words, offs[a], lens[a], strand[a], ops + (size_t)a * max_ops, n_ops[a], max_ops,
                                   begin[2 * a], begin[2 * a + 1], o, edits + 4 * (size_t)a);
        n_cigar[a] = o.n_cigar; md_len[a] = o.md_len;
    }
}

extern "C" void hh_finish(uint32_t bits, uint32_t big_endian, const uint32_t* genome, uint32_t genome_len, const uint32_t* read_words,
                          const uint32_t* offs, const uint32_t* lens, uint32_t n, const uint8_t* strand, const uint8_t* ops, uint32_t max_ops,
                          const uint32_t* n_ops, const uint32_t* begin, uint32_t* cigar, uint32_t max_cigar, uint32_t* n_cigar,
                          char* md, uint32_t max_md, uint32_t* md_len, uint32_t* edits)
{
#define HH_RUN(B, E) run<B, E>(genome, genome_len, read_words, offs, lens, n, strand, ops, max_ops, n_ops, begin, cigar, max_cigar, n_cigar, md, max_md, md_len, edits)
    if (bits == 2) { if (big_endian) HH_RUN(2, true); else HH_RUN(2, false); }
    else           { if (big_endian) HH_RUN(4, true); else HH_RUN(4, false); }
#undef HH_RUN
}
