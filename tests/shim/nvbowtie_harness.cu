// tests/shim/nvbowtie_harness.cu -- TEST INFRASTRUCTURE: a caller of nvBowtie's NON-template mapping entry points (boundary B-A2,
// nvBowtie/bowtie2/cuda/mapping.h: map_exact / map_approx / map / gather_ranges) written against nvBowtie's own PODs -- ReadsDef::type,
// FMIndexDef::type, PingPongQueuesView<uint32>, SeedHitDequeArray(DeviceView), ParamsPOD -- exactly as aligner_best_approx.h:150-240
// drives them.  This ONE object file is linked twice (oracle/ref_shim.mk):
//     nvbowtie_harness_ref    + nvBowtie's own mapping.cu, compiled where it lies (its sm_35-era kernels recompiled for sm_90a)
//     nvbowtie_harness_b200   + tests/shim/nvbowtie_mapping_b200.cu (include/nvbio_b200/shim/nvbowtie_mapping.h) + libnvbio_b200.so
// Both runs dump, per configuration: every read's deque size, its SeedHits in canonical (sorted) order, the range sizes in pop_top()
// order (which also proves that a valid priority deque was left behind), the reseed flags and gather_ranges' output.
#include <nvBowtie/bowtie2/cuda/defs.h>
#include <nvBowtie/bowtie2/cuda/mapping.h>
#include <nvbio/basic/numbers.h>
#include <nvbio/basic/priority_deque.h>
#include <nvbio/fmindex/bwt.h>
#include <nvbio/fmindex/ssa.h>
#include <thrust/device_vector.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using namespace nvbio;
using namespace nvbio::bowtie2::cuda;

// defined by the shim's replacement of mapping.cu (tests/shim/nvbowtie_mapping_b200.cu) only
extern "C" void nvbowtie_shim_calls(unsigned long long* mapped, unsigned long long* fallbacks) __attribute__((weak));

struct Rng
{
    uint64 s;
    explicit Rng(uint64 seed) : s( seed ) {}
    uint64 next() { s ^= s >> 12; s ^= s << 25; s ^= s >> 27; return s * 0x2545F4914F6CDD1Dull; }
    uint32 below(uint32 n) { return uint32( (next() >> 32) % n ); }
    double unit() { return double( next() >> 11 ) / 9007199254740992.0; }
};
template <typename T>
static void dump(const std::string& dir, const std::string& name, const std::vector<T>& v)
{
    const std::string path = dir + "/" + name;
    FILE* f = fopen( path.c_str(), "wb" );
    if (!f) { fprintf( stderr, "cannot write %s\n", path.c_str() ); exit( 2 ); }
    if (!v.empty()) fwrite( v.data(), sizeof(T), v.size(), f );
    fclose( f );
}
static void cuda_check(const char* what)
{
    cudaDeviceSynchronize();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { fprintf( stderr, "CUDA error after %s: %s\n", what, cudaGetErrorString( e ) ); exit( 3 ); }
}

// pop every deque from the top (smallest range first), as the select stage does: sizes in pop order
__global__ void pop_all_kernel(const uint32 n_reads, SeedHitDequeArrayDeviceView hits, uint32* sizes, const uint32 stride)
{
    const uint32 r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    typedef SeedHitDequeArrayDeviceView::hit_deque_type hit_deque_type;
    hit_deque_type deque = hits.get_deque( r );
    uint32 k = 0u;
    while (deque.size()) { sizes[ size_t(r) * stride + k++ ] = deque.top().get_range_size(); deque.pop_top(); }
}

int main(int argc, char** argv)
{
    if (argc < 2) { fprintf( stderr, "usage: nvbowtie_harness <outdir> [genome_len] [n_reads]\n" ); return 1; }
    const std::string out = argv[1];
    const uint32 genome_len = argc > 2 ? uint32( atoll( argv[2] ) ) : 400000u;
    const uint32 n_reads    = argc > 3 ? uint32( atoll( argv[3] ) ) : 4000u;
    Rng rng( 0x94D049BB133111EBull );

    // ---- genome with a few short repeat families, and its FM-index built by the reference's host code
    const uint32 genome_words = (genome_len + 15u) / 16u;
    std::vector<uint32> h_genome( genome_words + 4u, 0u );
    typedef PackedStream<uint32*,uint8,2u,true> host_stream;
    host_stream G( &h_genome[0] );
    for (uint32 i = 0; i < genome_len; ++i) G[i] = uint8( rng.below( 4u ) );
    for (uint32 fam = 0; fam < 40u; ++fam)                        // 40 families x 4 copies of a 300 bp unit
    {
        const uint32 src = rng.below( genome_len - 400u );
        for (uint32 c = 0; c < 3u; ++c)
        {
            const uint32 dst = rng.below( genome_len - 400u );
            for (uint32 j = 0; j < 300u; ++j) G[dst + j] = uint8( G[src + j] );
        }
    }
    {                                                             // a tandem repeat of an 11 bp unit over 5% of the genome: SA ranges ~1,800 rows wide
        const uint32 src = rng.below( genome_len / 2u ), span = genome_len / 20u;
        for (uint32 j = 11u; j < span; ++j) G[src + j] = uint8( G[src + j % 11u] );
    }
    std::vector<int32> h_sa( genome_len + 1u );
    gen_sa( genome_len, G, &h_sa[0] );
    std::vector<uint32> h_bwt( genome_words + 4u, 0u );
    host_stream B( &h_bwt[0] );
    const uint32 primary = gen_bwt_from_sa( genome_len, G, &h_sa[0], B );
    const uint32 n_blocks = (genome_len + 63u) / 64u;
    std::vector<uint32> h_occ( n_blocks * 4u + 4u, 0u ); uint32 cnt[4];
    build_occurrence_table<2u,64u>( PackedStream<const uint32*,uint8,2u,true>( &h_bwt[0] ), PackedStream<const uint32*,uint8,2u,true>( &h_bwt[0] ) + genome_len, &h_occ[0], cnt );
    std::vector<uint32> h_bwt_occ( n_blocks * 8u );
    for (uint32 k = 0; k < n_blocks; ++k)
        for (uint32 j = 0; j < 4u; ++j) { h_bwt_occ[ k*8u + j ] = h_bwt[ k*4u + j ]; h_bwt_occ[ k*8u + 4u + j ] = h_occ[ k*4u + j ]; }
    uint32 h_L2[5]; h_L2[0] = 0u; for (uint32 c = 0; c < 4u; ++c) h_L2[c+1] = h_L2[c] + cnt[c];
    const uint32 n_ssa = (genome_len + 16u) / 16u;
    std::vector<uint32> h_ssa( n_ssa );
    { SSA_index_multiple<16u> s( genome_len, (const uint32*)&h_sa[0] ); for (uint32 i = 0; i < n_ssa; ++i) h_ssa[i] = s.m_ssa[i]; h_ssa[0] = uint32(-1); }
    uint32 h_ct[256]; gen_bwt_count_table( h_ct );
    thrust::device_vector<uint32> d_bwt_occ( h_bwt_occ ), d_ssa( h_ssa ), d_L2( h_L2, h_L2 + 5 ), d_ct( h_ct, h_ct + 256 );
    typedef io::FMIndexDataDevice D;
    const D::bwt_occ_type bwt_occ_ptr( (const uint4*)thrust::raw_pointer_cast( d_bwt_occ.data() ) );
    const FMIndexDef::type fmi(
        genome_len, primary, thrust::raw_pointer_cast( d_L2.data() ),
        D::rank_dict_type( D::bwt_stream_type( D::bwt_type( bwt_occ_ptr ) ), D::occ_type( bwt_occ_ptr ), D::count_table_type( thrust::raw_pointer_cast( d_ct.data() ) ) ),
        D::ssa_type( D::ssa_ldg_type( thrust::raw_pointer_cast( d_ssa.data() ) ) ) );

    // ---- reads: DNA_N 4-bit big-endian, variable length, either strand, 2% substitutions, a few N's, a few very short reads
    std::vector<uint32> h_index( n_reads + 1u );
    std::vector<uint32> lens( n_reads );
    uint32 total = 0u, max_len = 0u;
    for (uint32 r = 0; r < n_reads; ++r) { lens[r] = (r % 13u == 5u) ? 10u + rng.below( 12u ) : 60u + rng.below( 91u ); total += lens[r]; max_len = nvbio::max( max_len, lens[r] ); }
    std::vector<uint32> h_reads( (total + 7u) / 8u + 4u, 0u );
    PackedStream<uint32*,uint8,4u,true> R( &h_reads[0] );
    std::vector<uint8> sym( 256 );
    uint32 cursor = 0u;
    for (uint32 r = 0; r < n_reads; ++r)
    {
        const uint32 len = lens[r];
        const uint32 pos = rng.below( genome_len - len - 1u );
        for (uint32 j = 0; j < len; ++j)
        {
            uint8 c = G[pos + j];
            const double u = rng.unit();
            if (u < 0.02)       c = uint8( (c + 1u + rng.below( 3u )) & 3u );
            else if (u < 0.023) c = 4u;
            sym[j] = c;
        }
        const bool flip = rng.below( 2u ) == 1u;
        h_index[r] = cursor;
        // nvBowtie keeps reads REVERSED in memory: the forward strand is searched by consuming the stored read front to back (mapping_inl.h:263-270)
        for (uint32 j = 0; j < len; ++j) R[cursor + len - 1u - j] = flip ? (sym[len-1u-j] < 4u ? 3u - sym[len-1u-j] : 4u) : sym[j];
        cursor += len;
    }
    h_index[n_reads] = cursor;
    thrust::device_vector<uint32> d_reads( h_reads ), d_index( h_index );
    io::SequenceDataInfo info;
    info.m_alphabet = DNA_N; info.m_n_seqs = n_reads; info.m_name_stream_len = 0u;
    info.m_sequence_stream_len = cursor; info.m_sequence_stream_words = uint32( h_reads.size() );
    info.m_has_qualities = 0u; info.m_min_sequence_len = 10u; info.m_max_sequence_len = max_len; info.m_avg_sequence_len = 100u;
    const ReadsDef::read_view_type view( info,
        ReadsDef::read_base_type( (const ReadsDef::read_storage_type*)thrust::raw_pointer_cast( d_reads.data() ) ),
        thrust::raw_pointer_cast( d_index.data() ), ReadsDef::read_qual_type( (const char*)NULL ), NULL, NULL );
    const ReadsDef::type reads( view );

    // ---- the input queue: most reads, shuffled
    std::vector<uint32> h_queue;
    for (uint32 r = 0; r < n_reads; ++r) if (r % 17u != 4u) h_queue.push_back( r );
    for (uint32 i = uint32( h_queue.size() ) - 1u; i > 0u; --i) std::swap( h_queue[i], h_queue[ rng.below( i + 1u ) ] );
    thrust::device_vector<uint32> d_queue( h_queue );
    nvbio::cuda::PingPongQueuesView<uint32> queues;
    queues.in_size = uint32( h_queue.size() ); queues.in_queue = thrust::raw_pointer_cast( d_queue.data() ); queues.out_size = NULL; queues.out_queue = NULL;

    struct Config { const char* name; int algo; uint32 seed_len, max_hits, subseed_len, retry, min_read_len; bool fw, rc; float k, m; };
    const Config configs[] = {
        { "exact_r0",   0, 22u, 100u,  0u, 0u, 20u, true,  true,  1.0f, 0.75f },      // nvBowtie --local defaults: seed interval 1 + 0.75 sqrt(len)
        { "exact_r1",   0, 20u, 100u,  0u, 1u, 20u, true,  true,  1.0f, 1.15f },      // end-to-end interval function, second reseeding round
        { "exact_fw",   0, 16u, 100u,  0u, 0u, 20u, true,  false, 1.0f, 0.75f },
        { "approx_r0",  1, 22u, 100u, 11u, 0u, 20u, true,  true,  1.0f, 0.75f },
        { "approx_rc",  1, 20u, 100u, 10u, 2u, 20u, false, true,  1.0f, 1.15f },
        { "map_sub",    2, 22u, 100u, 11u, 0u, 20u, true,  true,  1.0f, 0.75f },      // through map(): allow_sub with a subseed -> approximate
        { "map_nosub",  3, 22u, 100u,  0u, 0u, 20u, true,  true,  1.0f, 0.75f },      // through map(): no substitutions -> exact
        { "exact_tiny", 0, 12u,   6u,  0u, 0u, 20u, true,  true,  0.0f, 0.40f },      // short seeds, 6-slot deques: they overflow (sizes compared)
        // edges: one-slot deques; min_read_len above the seed length (reads of 60..69 bp are filtered, shorter ones too);
        // the NVB_MAP_MAX_PUSHES gate of map_approx (3 L + 1 ranges per seed): L = 33 is mapped by the shim, L = 34 falls back to
        // the reference's map_approx_t; map() with allow_sub and no subseed takes the reference's case pruning
        { "exact_h1",   0, 16u,   1u,  0u, 0u, 20u, true,  true,  1.0f, 0.75f },
        { "exact_min70",0, 16u, 100u,  0u, 1u, 70u, true,  true,  1.0f, 0.75f },
        { "approx_s33", 1, 33u, 100u, 16u, 0u, 20u, true,  true,  1.0f, 0.75f },
        { "approx_s34", 1, 34u, 100u, 17u, 1u, 20u, true,  true,  1.0f, 0.75f },
        { "approx_h1",  1, 14u,   1u,  7u, 2u, 20u, true,  true,  0.0f, 0.40f },
    };
    const uint32 n_configs = sizeof(configs) / sizeof(configs[0]);
    std::string json = "{\"program\": \"nvbowtie_mapping\", \"reads\": " + std::to_string( n_reads ) + ", \"queue\": " + std::to_string( h_queue.size() );
    for (uint32 c = 0; c < n_configs; ++c)
    {
        const Config& cfg = configs[c];
        ParamsPOD params;
        memset( &params, 0, sizeof(params) );
        params.seed_len = cfg.seed_len; params.seed_freq = SimpleFunc( SimpleFunc::SqrtFunc, cfg.k, cfg.m );
        params.max_hits = cfg.max_hits; params.max_reseed = 2u; params.rep_seeds = 4u; params.subseed_len = cfg.subseed_len; params.min_read_len = cfg.min_read_len;
        params.allow_sub = (cfg.algo == 1 || cfg.algo == 2) ? 1u : 0u;

        const uint32 arena = n_reads * cfg.max_hits;
        SeedHitDequeArray deques;
        deques.m_hits.resize( arena ); deques.m_counts.assign( n_reads, 0u ); deques.m_index.assign( n_reads, 0xFFFFFFFFu );
        deques.m_probs.resize( 2u * size_t(arena) + 1024u ); deques.m_probs_index.assign( n_reads, 0u );
        deques.m_pool.assign( 1u, 0u ); deques.m_probs_pool.assign( 1u, 0u );
        SeedHitDequeArrayDeviceView hits(
            nvbio::device_view( deques.m_counts ), nvbio::device_view( deques.m_index ), nvbio::device_view( deques.m_hits ),
            nvbio::device_view( deques.m_probs_index ), nvbio::device_view( deques.m_probs ), nvbio::device_view( deques.m_pool ), nvbio::device_view( deques.m_probs_pool ) );
        thrust::device_vector<uint8> d_reseed( h_queue.size(), uint8(9) );

        cudaEvent_t e0, e1; cudaEventCreate( &e0 ); cudaEventCreate( &e1 );
        cudaEventRecord( e0 );
        if (cfg.algo == 0)      map_exact ( reads, fmi, fmi, cfg.retry, queues, thrust::raw_pointer_cast( d_reseed.data() ), hits, params, cfg.fw, cfg.rc );
        else if (cfg.algo == 1) map_approx( reads, fmi, fmi, cfg.retry, queues, thrust::raw_pointer_cast( d_reseed.data() ), hits, params, cfg.fw, cfg.rc );
        else                    map       ( reads, fmi, fmi, cfg.retry, queues, thrust::raw_pointer_cast( d_reseed.data() ), hits, params, cfg.fw, cfg.rc );
        cudaEventRecord( e1 ); cudaEventSynchronize( e1 );
        float ms = 0.0f; cudaEventElapsedTime( &ms, e0, e1 );
        cuda_check( cfg.name );

        // canonical dumps
        std::vector<uint32> h_counts( n_reads ), h_hindex( n_reads ); std::vector<uint8> h_reseed( h_queue.size() );
        std::vector<uint64> h_hits( arena );
        cudaMemcpy( h_counts.data(), thrust::raw_pointer_cast( deques.m_counts.data() ), 4u * n_reads, cudaMemcpyDeviceToHost );
        cudaMemcpy( h_hindex.data(), thrust::raw_pointer_cast( deques.m_index.data() ),  4u * n_reads, cudaMemcpyDeviceToHost );
        cudaMemcpy( h_reseed.data(), thrust::raw_pointer_cast( d_reseed.data() ), h_queue.size(), cudaMemcpyDeviceToHost );
        cudaMemcpy( h_hits.data(), thrust::raw_pointer_cast( deques.m_hits.data() ), 8u * size_t(arena), cudaMemcpyDeviceToHost );
        std::vector<uint64> canon; std::vector<uint32> canon_sizes, empty_index; uint32 total_hits = 0u, overflowed = 0u;
        for (uint32 r = 0; r < n_reads; ++r)
        {
            std::vector<uint64> v;
            if (h_counts[r]) v.assign( h_hits.begin() + h_hindex[r], h_hits.begin() + h_hindex[r] + h_counts[r] );
            else             empty_index.push_back( h_hindex[r] );      // untouched (0xFFFFFFFF) unless a deque was allocated for the read
            std::sort( v.begin(), v.end() );
            canon.insert( canon.end(), v.begin(), v.end() );
            std::vector<uint32> sz; for (size_t i = 0; i < v.size(); ++i) sz.push_back( uint32( v[i] >> 32 ) & 0xFFFFFu );
            std::sort( sz.begin(), sz.end() );
            canon_sizes.insert( canon_sizes.end(), sz.begin(), sz.end() );
            total_hits += h_counts[r]; if (h_counts[r] == cfg.max_hits) ++overflowed;
        }
        // short reads keep the flag they had (the reference returns before writing it): normalise those entries
        for (size_t i = 0; i < h_queue.size(); ++i) if (lens[ h_queue[i] ] < params.min_read_len) h_reseed[i] = 9;
        dump( out, std::string( cfg.name ) + "_counts.bin", h_counts );
        dump( out, std::string( cfg.name ) + "_sizes.bin",  canon_sizes );
        dump( out, std::string( cfg.name ) + "_reseed.bin", h_reseed );
        dump( out, std::string( cfg.name ) + "_empty_index.bin", empty_index );
        if (cfg.max_hits >= 100u) dump( out, std::string( cfg.name ) + "_hits.bin", canon );

        // gather_ranges over an inclusive scan of the counts, then pop everything
        std::vector<uint32> h_scan( n_reads ); uint32 acc = 0u; for (uint32 r = 0; r < n_reads; ++r) { acc += h_counts[r]; h_scan[r] = acc; }
        thrust::device_vector<uint32> d_scan( h_scan ); thrust::device_vector<uint64> d_ranges( acc + 1u );
        if (acc) gather_ranges( acc, n_reads, hits, thrust::raw_pointer_cast( d_scan.data() ), thrust::raw_pointer_cast( d_ranges.data() ) );      // (the reference launches an empty grid for 0)
        cuda_check( "gather_ranges" );
        std::vector<uint64> h_ranges( acc ); if (acc) cudaMemcpy( h_ranges.data(), thrust::raw_pointer_cast( d_ranges.data() ), 8u * size_t(acc), cudaMemcpyDeviceToHost );
        uint64 range_total = 0u; for (size_t i = 0; i < h_ranges.size(); ++i) range_total += h_ranges[i];
        thrust::device_vector<uint32> d_pop( size_t(n_reads) * cfg.max_hits, 0u );
        pop_all_kernel<<< (n_reads + 127u) / 128u, 128u >>>( n_reads, hits, thrust::raw_pointer_cast( d_pop.data() ), cfg.max_hits );
        cuda_check( "pop_all" );
        std::vector<uint32> h_pop( d_pop.size() ); cudaMemcpy( h_pop.data(), thrust::raw_pointer_cast( d_pop.data() ), 4u * h_pop.size(), cudaMemcpyDeviceToHost );
        uint32 pop_order_ok = 1u;
        for (uint32 r = 0; r < n_reads; ++r) for (uint32 k = 1; k < h_counts[r]; ++k) if (h_pop[ size_t(r) * cfg.max_hits + k ] < h_pop[ size_t(r) * cfg.max_hits + k - 1u ]) pop_order_ok = 0u;
        dump( out, std::string( cfg.name ) + "_pop_sizes.bin", h_pop );
        char buf[512];
        snprintf( buf, sizeof(buf), ", \"%s\": {\"ms\": %.4f, \"hits\": %u, \"full_deques\": %u, \"range_total\": %llu, \"pop_order_ok\": %u}",
                  cfg.name, ms, total_hits, overflowed, (unsigned long long)range_total, pop_order_ok );
        json += buf;
    }
    unsigned long long mapped = 0u, fallbacks = 0u;
    if (nvbowtie_shim_calls) { nvbowtie_shim_calls( &mapped, &fallbacks ); json += ", \"shim\": 1"; }
    else json += ", \"shim\": 0";
    uint32 short_reads = 0u, below_seed = 0u;
    for (uint32 r = 0; r < n_reads; ++r) { short_reads += lens[r] < 20u; below_seed += lens[r] < 22u; }
    json += ", \"reads_below_20\": " + std::to_string( short_reads ) + ", \"reads_below_22\": " + std::to_string( below_seed );
    json += ", \"b200_calls\": {\"mapped\": " + std::to_string( mapped ) + ", \"fallbacks\": " + std::to_string( fallbacks ) + "}}";
    printf( "%s\n", json.c_str() );
    return 0;
}
