// oracle/ref_mapq_paired.cpp -- TEST INFRASTRUCTURE (oracle/_ref/libnvbio_ref_mapq_paired.so, built by oracle/ref_mapq_paired.mk):
// nvBowtie's OWN BowtieMapq2 on PAIRED best alignments, compiled from an nvbio source tree where it lies, so that the paired MAPQ of
// nvb_seed_extend_paired_mapq is pinned against the reference's code instead of a model of it.
#include <nvbio/basic/types.h>
#include <nvBowtie/bowtie2/cuda/mapq.h>
#include <nvbio/io/alignments.h>
#include <omp.h>

using namespace nvbio;

namespace {
// the three members BowtieMapq2 reads from a scoring scheme (perfect_score, min_score, m_monotone; scoring.h:272-281,347), with each
// mate's minimum score given as a number instead of a SimpleFunc of its length (a --score-min function gives equal lengths equal values,
// so the look-up by length is exact)
struct MapqModelSchemePE
{
    int32  m_match_bonus, m_min1, m_min2;
    uint32 m_len1;
    bool   m_monotone;
    int32 perfect_score(const uint32 read_len) const { return int32(read_len) * m_match_bonus; }
    int32 min_score(const uint32 read_len) const { return read_len == m_len1 ? m_min1 : m_min2; }
};
} // anonymous namespace

extern "C" {

// nvBowtie's BowtieMapq2 of a PAIRED best alignment (mapq.h:155-170 with is_paired()), as MapqFunctorPE runs it
// (aligner_best_approx_paired.h:50-96): the best pair is (a1 = mate 1 of score s1, o1 = mate 2 of score s2), both flagged paired; the
// second is none (kind 0), a paired second (kind 1: a2 / o2 of scores t1 / t2, both flagged paired) or an unpaired second (kind 2: a2
// of score t1 without the paired flag).  Mate 1 has length len1 and minimum score min1, mate 2 len2 / min2.  The reference sums the
// per-mate scores itself (io::Alignment keeps 17 bits and a sign per score).
void ref_nvbowtie_mapq_paired(const int32* s1, const int32* s2, const uint8* kind, const int32* t1, const int32* t2, const uint32* len1,
                              const uint32* len2, const int32* match_bonus, const int32* min1, const int32* min2, uint32 n, uint8* mapq)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        MapqModelSchemePE sc; sc.m_match_bonus = match_bonus[i]; sc.m_min1 = min1[i]; sc.m_min2 = min2[i]; sc.m_len1 = len1[i];
        sc.m_monotone = (match_bonus[i] == 0);
        const bowtie2::cuda::BowtieMapq2<MapqModelSchemePE> eval( sc );
        const io::Alignment a1( 0u, 0u, s1[i], 0u, 0u, true );
        const io::Alignment o1( 500u, 0u, s2[i], 1u, 1u, true );
        const io::Alignment a2 = kind[i] == 0 ? io::Alignment::invalid() : io::Alignment( 1000u, 0u, t1[i], 0u, 0u, kind[i] == 1 );
        const io::Alignment o2 = kind[i] == 1 ? io::Alignment( 1500u, 0u, t2[i], 1u, 1u, true ) : io::Alignment::invalid();
        const io::BestPairedAlignments best( io::BestAlignments( a1, a2 ), io::BestAlignments( o1, o2 ) );
        mapq[i] = uint8( eval( best, best.anchor_mate<0>() ? len2[i] : len1[i], best.anchor_mate<0>() ? len1[i] : len2[i] ) );
    }
}

} // extern "C"
