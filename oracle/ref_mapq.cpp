// oracle/ref_mapq.cpp -- TEST INFRASTRUCTURE (oracle/_ref/libnvbio_ref_mapq.so, built by oracle/ref_mapq.mk): nvBowtie's OWN
// BowtieMapq2 and SimpleFunc, compiled from an nvbio source tree where it lies, so that the MAPQ of nvb_seed_extend_mapq and the
// host-evaluated --score-min table of nvbio_b200.MapqParams are pinned against the reference's code instead of a model of it.
#include <nvbio/basic/types.h>
#include <nvBowtie/bowtie2/cuda/func.h>
#include <nvBowtie/bowtie2/cuda/mapq.h>
#include <nvbio/io/alignments.h>
#include <omp.h>

using namespace nvbio;

namespace {
// the three members BowtieMapq2 reads from a scoring scheme (perfect_score, min_score, m_monotone; scoring.h:272-281,347), with the
// minimum score given as a number instead of a SimpleFunc -- the way TableGotohScheme (ref_shim.cpp) models a scheme
struct MapqModelScheme
{
    int32 m_match_bonus, m_min;
    bool  m_monotone;
    int32 perfect_score(const uint32 read_len) const { return int32(read_len) * m_match_bonus; }
    int32 min_score(const uint32) const { return m_min; }
};
} // anonymous namespace

extern "C" {

// nvBowtie's BowtieMapq2 (mapq.h:142-331) of unpaired reads, as aligner_best_approx.h:291-305 runs it: mapq[i] for a best alignment of
// score best[i], a second one of score second[i] when has_second[i], a read of length len[i] and a scheme with match bonus match_bonus[i]
// (monotone when 0, scoring_inl.h:144) and minimum score min_score[i]
void ref_nvbowtie_mapq(const int32* best, const uint8* has_second, const int32* second, const uint32* len, const int32* match_bonus,
                       const int32* min_score, uint32 n, uint8* mapq)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        MapqModelScheme sc; sc.m_match_bonus = match_bonus[i]; sc.m_min = min_score[i]; sc.m_monotone = (match_bonus[i] == 0);
        const bowtie2::cuda::BowtieMapq2<MapqModelScheme> eval( sc );
        const io::Alignment a1( 0u, 0u, best[i], 0u );
        const io::Alignment a2 = has_second[i] ? io::Alignment( 1u, 0u, second[i], 0u ) : io::Alignment::invalid();
        mapq[i] = uint8( eval( io::BestPairedAlignments( io::BestAlignments( a1, a2 ) ), len[i], 0u ) );
    }
}

// nvBowtie's SimpleFunc (func.h:39-51), type 0 linear, 1 log, 2 sqrt: out[i] = f(x[i])
void ref_nvbowtie_simple_func(int type, float k, float m, const int32* x, uint32 n, int32* out)
{
    const bowtie2::cuda::SimpleFunc f( bowtie2::cuda::SimpleFunc::Type( type ), k, m );
    for (uint32 i = 0; i < n; ++i)
        out[i] = f( x[i] );
}

} // extern "C"
