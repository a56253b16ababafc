// tests/shim/nvbowtie_score_harness.cu -- TEST INFRASTRUCTURE: nvBowtie's best-score extension stage (boundary B-B2) driven through
// nvBowtie's own template detail::banded_score_best(band_len, pipeline, aligner, params) (score_best_inl.h:154-200) -- the body of
// score_best_t / score_best (:212-234) -- with nvBowtie's types: a DNA_N read batch WITH base qualities (ReadsDef::type), the 2-bit genome
// stream, HitQueues (read_id / seed / loc / score / sink), io::Alignment best-alignment records, SmithWatermanScoringScheme<> (its
// --local preset and the end-to-end default) and ParamsPOD.  The pipeline object is a POD with the member names the stream reads
// (pipeline_states.h:59-170); nvBowtie's own needs its whole Aligner to be constructed.
// Compiled twice: as is (reference kernels) and with -DNVBIO_B200_SHIM (include/nvbio_b200/shim/nvbowtie_scoring.h + libnvbio_b200.so);
// both dump hit.score / hit.sink of every queued hit.
#include <nvBowtie/bowtie2/cuda/defs.h>
#include <nvbio/alignment/alignment.h>
#include <nvbio/alignment/batched.h>
#include <nvBowtie/bowtie2/cuda/reads_def.h>
#include <nvBowtie/bowtie2/cuda/scoring.h>
#include <nvBowtie/bowtie2/cuda/scoring_queues.h>
#include <nvBowtie/bowtie2/cuda/score_best_inl.h>
#if defined(NVBIO_B200_SHIM)
#include <nvbio_b200/shim/nvbowtie_scoring.h>
#endif
#include <thrust/device_vector.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace harness {
using namespace nvbio;
using namespace nvbio::bowtie2::cuda;

struct Rng
{
    uint64 s;
    explicit Rng(uint64 seed) : s( seed ) {}
    uint64 next() { s ^= s >> 12; s ^= s << 25; s ^= s >> 27; return s * 0x2545F4914F6CDD1Dull; }
    uint32 below(uint32 n) { return uint32( (next() >> 32) % n ); }
    double unit() { return double( next() >> 11 ) / 9007199254740992.0; }
};
template <typename T>
static void dump(const std::string& dir, const std::string& name, const thrust::device_vector<T>& d)
{
    std::vector<T> h( d.size() );
    if (!h.empty()) cudaMemcpy( h.data(), thrust::raw_pointer_cast( d.data() ), sizeof(T) * h.size(), cudaMemcpyDeviceToHost );
    const std::string path = dir + "/" + name;
    FILE* f = fopen( path.c_str(), "wb" );
    if (!f) { fprintf( stderr, "cannot write %s\n", path.c_str() ); exit( 2 ); }
    if (!h.empty()) fwrite( h.data(), sizeof(T), h.size(), f );
    fclose( f );
}

typedef SmithWatermanScoringScheme<>    scheme_t;

// the members of BestApproxScoringPipelineState<scheme> that BestScoreStream / AlignmentStrings touch (pipeline_states.h:59-170)
struct HarnessPipeline
{
    typedef ReadsDef::type                                                      read_batch_type;
    typedef PackedStream<nvbio::cuda::ldg_pointer<uint32>,uint8,2u,true>        genome_iterator;
    typedef scheme_t                                                            scheme_type;
    struct Queues { HitQueuesDeviceView hits; };

    read_batch_type     reads, reads_o;
    uint32              genome_length;
    genome_iterator     genome;
    Queues              scoring_queues;
    uint32              hits_queue_size;
    uint32*             idx_queue;
    uint8*              dp_buffer;
    uint64              dp_buffer_size;
    scheme_t            scoring_scheme;
    int32               score_limit;
    io::Alignment*      best_alignments;
    uint32              best_stride;

    HarnessPipeline(const read_batch_type r, const genome_iterator g) : reads( r ), reads_o( r ), genome( g ) {}
};

int run(int argc, char** argv)
{
    if (argc < 2) { fprintf( stderr, "usage: nvbowtie_score_harness <outdir> [genome_len] [n_reads] [n_hits]\n" ); return 1; }
    const std::string out = argv[1];
    const uint32 genome_len = argc > 2 ? uint32( atoll( argv[2] ) ) : 2000000u;
    const uint32 n_reads    = argc > 3 ? uint32( atoll( argv[3] ) ) : 20000u;
    const uint32 n_hits     = argc > 4 ? uint32( atoll( argv[4] ) ) : 100000u;
    Rng rng( 0x2545F4914F6CDD1Dull );

    const uint32 genome_words = (genome_len + 15u) / 16u;
    std::vector<uint32> h_genome( genome_words + 8u, 0u );
    PackedStream<uint32*,uint8,2u,true> G( &h_genome[0] );
    for (uint32 i = 0; i < genome_len; ++i) G[i] = uint8( rng.below( 4u ) );
    thrust::device_vector<uint32> d_genome( h_genome );

    // reads with qualities: nvBowtie keeps them REVERSED in memory (the loaders flip them back, alignment_utils.h:205-212)
    std::vector<uint32> h_index( n_reads + 1u ), lens( n_reads ), origin( n_reads );
    uint32 total = 0u, max_len = 0u;
    for (uint32 r = 0; r < n_reads; ++r) { lens[r] = 50u + rng.below( 101u ); total += lens[r]; max_len = nvbio::max( max_len, lens[r] ); }
    std::vector<uint32> h_reads( (total + 7u) / 8u + 4u, 0u );
    std::vector<char>   h_quals( total + 16u, 0 );
    PackedStream<uint32*,uint8,4u,true> R( &h_reads[0] );
    uint32 cursor = 0u;
    std::vector<uint8> sym( 256 );
    for (uint32 r = 0; r < n_reads; ++r)
    {
        const uint32 len = lens[r];
        const uint32 pos = 20u + rng.below( genome_len - len - 60u );
        origin[r] = pos;
        for (uint32 j = 0; j < len; ++j)
        {
            uint8 c = G[pos + j];
            const double u = rng.unit();
            if (u < 0.03)       c = uint8( (c + 1u + rng.below( 3u )) & 3u );
            else if (u < 0.034) c = 4u;
            sym[j] = c;
        }
        if (rng.below( 50u ) == 0u && len > 60u) { for (uint32 j = 30u; j + 2u < len; ++j) sym[j] = sym[j + 2u]; }     // a 2-base deletion
        if (r % 211u == 17u) for (uint32 j = 0; j < len; ++j) sym[j] = 4u;                                              // all-N reads
        // base qualities: uniform in 0..44, or the whole read at 0, or the whole read at 40 or more
        const uint32 qmode = r % 29u == 5u ? 1u : r % 29u == 11u ? 2u : 0u;
        h_index[r] = cursor;
        for (uint32 j = 0; j < len; ++j)                                                                                  // stored reversed
        {
            R[cursor + j] = sym[len - 1u - j];
            h_quals[cursor + j] = char( qmode == 1u ? 0u : qmode == 2u ? 40u + rng.below( 10u ) : rng.below( 45u ) );
        }
        cursor += len;
    }
    h_index[n_reads] = cursor;
    thrust::device_vector<uint32> d_reads( h_reads ), d_index( h_index );
    thrust::device_vector<char>   d_quals( h_quals );
    io::SequenceDataInfo info;
    info.m_alphabet = DNA_N; info.m_n_seqs = n_reads; info.m_name_stream_len = 0u;
    info.m_sequence_stream_len = cursor; info.m_sequence_stream_words = uint32( h_reads.size() );
    info.m_has_qualities = 1u; info.m_min_sequence_len = 50u; info.m_max_sequence_len = max_len; info.m_avg_sequence_len = 100u;
    const ReadsDef::read_view_type view( info,
        ReadsDef::read_base_type( (const ReadsDef::read_storage_type*)thrust::raw_pointer_cast( d_reads.data() ) ),
        thrust::raw_pointer_cast( d_index.data() ), ReadsDef::read_qual_type( (const char*)thrust::raw_pointer_cast( d_quals.data() ) ), NULL, NULL );
    const ReadsDef::type reads( view );

    // the hit queue: read, strand flag, located position (near the read's origin on the forward strand, anywhere on the other), sorting index
    std::vector<uint32> h_read_id( n_hits ), h_loc( n_hits ), h_idx( n_hits );
    std::vector<packed_seed> h_seed( n_hits );
    for (uint32 h = 0; h < n_hits; ++h)
    {
        const uint32 r = rng.below( n_reads );
        h_read_id[h] = r;
        packed_seed s; s.pos_in_read = 0u; s.index_dir = 0u; s.rc = rng.below( 4u ) == 0u ? 1u : 0u; s.top_flag = 0u;
        h_seed[h] = s;
        const int32 jitter = int32( rng.below( 21u ) ) - 10;
        h_loc[h] = (h % 97u == 0u) ? rng.below( 40u )                                   // windows clamped at the genome start ...
                 : (h % 89u == 0u) ? genome_len - rng.below( 100u ) - 1u               // ... and at its end
                 : uint32( int32( origin[r] ) + jitter );
        h_idx[h] = h;
    }
    for (uint32 i = n_hits - 1u; i > 0u; --i) std::swap( h_idx[i], h_idx[ rng.below( i + 1u ) ] );
    thrust::device_vector<uint32> d_read_id( h_read_id ), d_loc( h_loc ), d_idx( h_idx ), d_ssa( n_hits, 0u ), d_sink( n_hits, 0u ), d_osink( 1 );
    thrust::device_vector<packed_seed> d_seed( h_seed );
    thrust::device_vector<int32> d_score( n_hits, 0 ), d_oscore( 1 );
    thrust::device_vector<uint32> d_oloc( 1 );
    const HitQueuesDeviceView hits_view(
        nvbio::device_view( d_read_id ), nvbio::device_view( d_seed ), nvbio::device_view( d_ssa ), nvbio::device_view( d_loc ),
        nvbio::device_view( d_score ), nvbio::device_view( d_sink ), nvbio::device_view( d_oloc ), nvbio::device_view( d_oscore ),
        nvbio::device_view( d_osink ), nvbio::device_view( d_oscore ), nvbio::device_view( d_osink ) );

    std::vector<io::Alignment> h_best( 2u * n_reads, io::Alignment( 0u, 0u, io::Alignment::min_score(), 0u ) );
    thrust::device_vector<io::Alignment> d_best( h_best );
    thrust::device_vector<uint8> d_dp( 64u << 20 );

    std::string json = "{\"program\": \"nvbowtie_score_best\", \"hits\": " + std::to_string( n_hits );
    // every band banded_score_best dispatches to (3, 7, 15, 31), --local and end-to-end
    const char* names[7] = { "local_b31", "local_b15", "e2e_b31", "e2e_b7", "local_b3", "local_b7", "e2e_b15" };
    const bool   is_local[7] = { true, true, false, false, true, true, false };
    const uint32 bands[7]    = { 31u, 15u, 31u, 7u, 3u, 7u, 15u };
    for (uint32 c = 0; c < 7u; ++c)
    {
        const bool local = is_local[c];
        const uint32 band_len = bands[c];
        HarnessPipeline pipeline( reads, HarnessPipeline::genome_iterator( nvbio::cuda::ldg_pointer<uint32>( thrust::raw_pointer_cast( d_genome.data() ) ) ) );
        pipeline.genome_length = genome_len;
        pipeline.scoring_queues.hits = hits_view;
        pipeline.hits_queue_size = n_hits; pipeline.idx_queue = thrust::raw_pointer_cast( d_idx.data() );
        pipeline.dp_buffer = thrust::raw_pointer_cast( d_dp.data() ); pipeline.dp_buffer_size = d_dp.size();
        pipeline.scoring_scheme = local ? scheme_t::local() : scheme_t();
        // min_score = max(second best, score_limit) has no effect here: banded_score_best runs the thread scheduler, whose single pass
        // ends at the last pattern row, and the reference checks min_score only after a window that ends before it (gotoh_banded_inl.h:
        // 622-633).  A min_score in reach is pinned where it matters, on the staged scheduler (shim_harness edges)
        pipeline.score_limit = -1000;
        pipeline.best_alignments = thrust::raw_pointer_cast( d_best.data() ); pipeline.best_stride = n_reads;
        ParamsPOD params; memset( &params, 0, sizeof(params) );
        params.alignment_type = local ? LocalAlignment : EndToEndAlignment;
        thrust::fill( d_score.begin(), d_score.end(), 12345 ); thrust::fill( d_sink.begin(), d_sink.end(), 54321u );

        cudaEvent_t e0, e1; cudaEventCreate( &e0 ); cudaEventCreate( &e1 );
        float best_ms = 1e30f;
        for (int rep = 0; rep < 3; ++rep)
        {
            cudaEventRecord( e0 );
            if (local) detail::banded_score_best( band_len, pipeline, pipeline.scoring_scheme.local_aligner(), params );
            else       detail::banded_score_best( band_len, pipeline, pipeline.scoring_scheme.end_to_end_aligner(), params );
            cudaEventRecord( e1 ); cudaEventSynchronize( e1 );
            float ms; cudaEventElapsedTime( &ms, e0, e1 ); if (rep && ms < best_ms) best_ms = ms;
        }
        cudaDeviceSynchronize();
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { fprintf( stderr, "CUDA error in %s: %s\n", names[c], cudaGetErrorString( e ) ); return 3; }
        dump( out, std::string( names[c] ) + "_score.bin", d_score );
        {   // how many hits the worst_score clamp decided (no alignment in the window, or a score below the scheme's worst)
            std::vector<int32> h( n_hits ); cudaMemcpy( h.data(), thrust::raw_pointer_cast( d_score.data() ), 4u * n_hits, cudaMemcpyDeviceToHost );
            uint32 clamped = 0u; for (uint32 i = 0; i < n_hits; ++i) clamped += h[i] == scheme_t::worst_score;
            json += ", \"" + std::string( names[c] ) + "_clamped\": " + std::to_string( clamped );
        }
        dump( out, std::string( names[c] ) + "_sink.bin",  d_sink );
        char buf[256];
        snprintf( buf, sizeof(buf), ", \"%s_ms\": %.4f", names[c], best_ms ); json += buf;
    }
#if defined(NVBIO_B200_SHIM)
    { const nvbio::b200::shim_stats& st = nvbio::b200::stats();
      json += ", \"shim\": 1, \"b200_calls\": {\"banded\": " + std::to_string( st.banded_score ) + ", \"fallbacks\": " + std::to_string( st.fallbacks ) + "}"; }
#else
    json += ", \"shim\": 0";
#endif
    json += "}";
    printf( "%s\n", json.c_str() );
    return 0;
}

} // namespace harness

int main(int argc, char** argv) { return harness::run( argc, argv ); }
