// oracle/ref_finish.cpp -- TEST INFRASTRUCTURE (oracle/_ref/libnvbio_ref_finish.so, built by oracle/ref_finish.mk): nvbio's OWN output
// helpers io::analyze_md_string, io::count_symbols and io::reference_cigar_length (nvbio/io/output/output_utils.h:42-121), compiled from an
// nvbio source tree where they lie, so that the XM / XO / XG, indel totals and genome spans of nvb_finish_alignments are pinned against
// the reference's code instead of a model of it.
#include <nvbio/basic/types.h>
#include <nvbio/io/alignments.h>
#include <nvbio/io/output/output_utils.h>
#include <vector>

using namespace nvbio;

extern "C" {

// n alignments: MDS vector i = mds[mds_off[i], mds_off[i + 1]) (nvBowtie's layout, two length bytes first); io::Cigar vector i = the
// (type, length) pairs cigar[2 * cigar_off[i], 2 * cigar_off[i + 1]) in nvBowtie's storage order (END -> START).  out[6 i ..] = n_mm,
// n_gapo, n_gape of analyze_md_string, count_symbols(INSERTION), count_symbols(DELETION), reference_cigar_length.
void ref_finish_analyze(const uint8* mds, const uint64* mds_off, const uint16* cigar, const uint64* cigar_off, uint32 n, uint32* out)
{
    for (uint32 i = 0; i < n; ++i)
    {
        uint32 mm = 0, gapo = 0, gape = 0;
        io::analyze_md_string( mds + mds_off[i], mm, gapo, gape );
        const uint32 len = uint32( cigar_off[i + 1] - cigar_off[i] );
        std::vector<io::Cigar> c( len );
        for (uint32 k = 0; k < len; ++k)
            c[k] = io::Cigar( uint8( cigar[2 * (cigar_off[i] + k)] ), cigar[2 * (cigar_off[i] + k) + 1] );
        out[6 * i + 0] = mm;
        out[6 * i + 1] = gapo;
        out[6 * i + 2] = gape;
        out[6 * i + 3] = io::count_symbols( io::Cigar::INSERTION, &c[0], len );
        out[6 * i + 4] = io::count_symbols( io::Cigar::DELETION, &c[0], len );
        out[6 * i + 5] = io::reference_cigar_length( &c[0], len );
    }
}

} // extern "C"
