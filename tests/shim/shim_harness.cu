// tests/shim/shim_harness.cu -- TEST INFRASTRUCTURE: programs written against NVBIO'S OWN TYPES, compiled twice from this one
// source against the reference headers where they lie (/root/reference):
//
//     shim_harness_ref    plain reference: nvbio's templates and its own sm_35-era kernels, recompiled for sm_90a
//     shim_harness_b200   the same source with -DNVBIO_B200_SHIM: <nvbio_b200/shim/nvbio_shim.h> is included after nvbio's
//                         headers and libnvbio_b200.so is linked -- nothing else changes
//
// and run on the same deterministic inputs; every result array is dumped so that the two runs can be compared bit for bit
// (tests/test_gpu_shim.py; oracle/ref_shim.mk builds both).  Three programs (the third, edges, is described at run_edges):
//
//   fmmap <outdir> [genome_len] [n_reads] [read_len]
//       the seed -> rank -> locate -> diagonal -> window -> banded DP -> best-per-read loop of nvbio's fmmap example
//       (examples/fmmap/fmmap.cu:255-400), on io::FMIndexDataDevice::fm_index_type, io::SequenceDataAccess<DNA_N> reads
//       (4-bit, forward + reverse-complement strings), InfixSet seeds, FMIndexFilterDevice::rank/locate, SparseStringSet
//       infixes and aln::batch_banded_alignment_score<31> with a LOCAL Gotoh aligner and BestSink<int16> / BestSink<int32>.
//   batch <outdir> [n_tasks]
//       the batch scoring test of nvbio-test/alignment_test.cu:532-585: a user-defined alignment stream (4-bit little-endian
//       patterns, 2-bit little-endian texts, int16 scores) driven through BatchedBandedAlignmentScore<BAND_LEN,stream,
//       DeviceThreadScheduler / DeviceStagedThreadScheduler>::enact for GLOBAL / SEMI_GLOBAL / LOCAL Gotoh, plus
//       aln::batch_alignment_score (full matrix) over packed string sets.
#include <nvbio/basic/types.h>
#include <nvbio/basic/numbers.h>
#include <nvbio/basic/packedstream.h>
#include <nvbio/basic/packedstream_loader.h>
#include <nvbio/basic/vector_view.h>
#include <nvbio/basic/vector.h>
#include <nvbio/basic/cuda/ldg.h>
#include <nvbio/strings/string_set.h>
#include <nvbio/strings/infix.h>
#include <nvbio/fmindex/bwt.h>
#include <nvbio/fmindex/ssa.h>
#include <nvbio/fmindex/fmindex.h>
#include <nvbio/fmindex/filter.h>
#include <nvbio/io/fmindex/fmindex.h>
#include <nvbio/io/sequence/sequence.h>
#include <nvbio/io/sequence/sequence_access.h>
#include <nvbio/alignment/alignment.h>
#include <nvbio/alignment/batched.h>
#include <thrust/device_vector.h>
#include <thrust/host_vector.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#if defined(NVBIO_B200_SHIM)
#include <nvbio_b200/shim/nvbio_shim.h>
#endif

using namespace nvbio;

// ---------------------------------------------------------------------------------------------------
// utilities
// ---------------------------------------------------------------------------------------------------
struct Rng
{
    uint64 s;
    explicit Rng(uint64 seed) : s( seed ) {}
    uint64 next() { s ^= s >> 12; s ^= s << 25; s ^= s >> 27; return s * 0x2545F4914F6CDD1Dull; }
    uint32 below(uint32 n) { return uint32( (next() >> 32) % n ); }
    double unit() { return double( next() >> 11 ) / 9007199254740992.0; }
};

template <typename T>
static void dump(const std::string& dir, const char* name, const T* p, size_t n)
{
    const std::string path = dir + "/" + name;
    FILE* f = fopen( path.c_str(), "wb" );
    if (!f) { fprintf( stderr, "cannot write %s\n", path.c_str() ); exit( 2 ); }
    fwrite( p, sizeof(T), n, f );
    fclose( f );
}
template <typename T>
static void dump(const std::string& dir, const char* name, const thrust::device_vector<T>& d, size_t n)
{
    std::vector<T> h( n );
    if (n) cudaMemcpy( h.data(), thrust::raw_pointer_cast( d.data() ), sizeof(T) * n, cudaMemcpyDeviceToHost );
    dump( dir, name, h.data(), n );
}
static void cuda_check(const char* what)
{
    cudaDeviceSynchronize();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { fprintf( stderr, "CUDA error after %s: %s\n", what, cudaGetErrorString( e ) ); exit( 3 ); }
}
struct GpuTimer
{
    cudaEvent_t a, b;
    GpuTimer()  { cudaEventCreate( &a ); cudaEventCreate( &b ); }
    void start() { cudaEventRecord( a ); }
    float stop() { cudaEventRecord( b ); cudaEventSynchronize( b ); float ms; cudaEventElapsedTime( &ms, a, b ); return ms; }
};

// ---------------------------------------------------------------------------------------------------
// program 1: fmmap
// ---------------------------------------------------------------------------------------------------
typedef io::FMIndexDataDevice::fm_index_type                        fm_index_type;
typedef FMIndexFilterDevice<fm_index_type>                          fm_filter_type;
typedef io::SequenceDataAccess<DNA_N>                               read_access_type;
typedef io::SequenceDataAccess<DNA>                                 genome_access_type;

// (index-pos, seed-id) -> diagonal (text-pos of the read's first base, string id)
__global__ void hits_to_diagonals_kernel(const uint32 n, uint2* hits, const string_set_infix_coord_type* seeds)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint2 hit = hits[i];
    const string_set_infix_coord_type seed = seeds[ hit.y ];
    hits[i] = make_uint2( hit.x - infix_begin( seed ), string_id( seed ) );
}
// per diagonal: the read's range in the read stream and the genome window the band covers (examples/fmmap/fmmap.cu:190-208)
template <uint32 BAND_LEN>
__global__ void infixes_kernel(const uint32 n, const uint2* diagonals, const io::ConstSequenceDataView reads_view, const uint32 genome_len,
                               string_infix_coord_type* read_infixes, string_infix_coord_type* genome_infixes)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const read_access_type reads( reads_view );
    const uint2  d          = diagonals[i];
    const uint2  read_range = reads.get_range( d.y );
    const uint32 read_len   = read_range.y - read_range.x;
    const uint32 text_pos   = d.x;
    const uint32 g_begin    = text_pos > BAND_LEN/2 ? text_pos - BAND_LEN/2 : 0u;
    const uint32 g_end      = nvbio::min( g_begin + read_len + BAND_LEN, genome_len );
    read_infixes[i]   = read_range;
    genome_infixes[i] = make_uint2( g_begin, g_end );
}
template <typename sink_type>
__global__ void best_per_read_kernel(const uint32 n, const uint2* diagonals, const sink_type* sinks, int32* best)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    atomicMax( best + diagonals[i].y / 2u, int32( sinks[i].score ) );       // strings 2r, 2r+1 = the two strands of read r
}
template <typename sink_type>
__global__ void split_sinks_kernel(const uint32 n, const sink_type* sinks, int32* score, uint2* sink)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    score[i] = int32( sinks[i].score ); sink[i] = sinks[i].sink;
}

template <typename score_type>
static float extend_hits(const char* tag, const std::string& out, const uint32 n_hits, const uint32 n_reads, const uint32 max_read_len,
                         const thrust::device_vector<uint2>& diagonals,
                         const thrust::device_vector<string_infix_coord_type>& read_infix_coords,
                         const thrust::device_vector<string_infix_coord_type>& genome_infix_coords,
                         const read_access_type& reads_access, const genome_access_type& genome_access)
{
    typedef aln::BestSink<score_type>                                       sink_type;
    typedef read_access_type::sequence_stream_type                          read_stream;
    typedef genome_access_type::sequence_stream_type                        genome_stream;
    typedef const string_infix_coord_type*                                  infix_iterator;
    static const uint32 BAND_LEN = 31u;

    thrust::device_vector<sink_type> sinks( n_hits );
    const SparseStringSet<read_stream,infix_iterator>   read_infix_set( n_hits, reads_access.sequence_stream(), thrust::raw_pointer_cast( read_infix_coords.data() ) );
    const SparseStringSet<genome_stream,infix_iterator> genome_infix_set( n_hits, genome_access.sequence_stream(), thrust::raw_pointer_cast( genome_infix_coords.data() ) );
    const aln::SimpleGotohScheme gotoh( 2, -2, -5, -3 );

    GpuTimer timer; float best_ms = 1e30f;
    for (int rep = 0; rep < 3; ++rep)
    {
        timer.start();
        aln::batch_banded_alignment_score<BAND_LEN>(
            aln::make_gotoh_aligner<aln::LOCAL>( gotoh ),
            read_infix_set,
            genome_infix_set,
            thrust::raw_pointer_cast( sinks.data() ),
            aln::DeviceThreadScheduler(),
            max_read_len,
            max_read_len + BAND_LEN );
        const float ms = timer.stop();
        if (rep && ms < best_ms) best_ms = ms;
    }
    cuda_check( "batch_banded_alignment_score" );

    thrust::device_vector<int32> score( n_hits ), best( n_reads, -1000000 );
    thrust::device_vector<uint2> sink( n_hits );
    const uint32 grid = (n_hits + 255u) / 256u;
    split_sinks_kernel<<<grid,256>>>( n_hits, thrust::raw_pointer_cast( sinks.data() ), thrust::raw_pointer_cast( score.data() ), thrust::raw_pointer_cast( sink.data() ) );
    best_per_read_kernel<<<grid,256>>>( n_hits, thrust::raw_pointer_cast( diagonals.data() ), thrust::raw_pointer_cast( sinks.data() ), thrust::raw_pointer_cast( best.data() ) );
    cuda_check( "best_per_read" );
    dump( out, (std::string("fmmap_scores_") + tag + ".bin").c_str(), score, n_hits );
    dump( out, (std::string("fmmap_sinks_") + tag + ".bin").c_str(), sink, n_hits );
    dump( out, (std::string("fmmap_best_") + tag + ".bin").c_str(), best, n_reads );
    return best_ms;
}

static int run_fmmap(const std::string& out, const uint32 genome_len, const uint32 n_reads, const uint32 read_len)
{
    static const uint32 SEED_LEN = 22u, SEED_INTV = 10u, BAND_LEN = 31u;
    Rng rng( 0x9E3779B97F4A7C15ull );

    // ---- genome (2-bit big-endian, the io::SequenceData<DNA> layout) and its FM-index, built with the reference's own host code
    const uint32 genome_words = (genome_len + 15u) / 16u;
    std::vector<uint32> h_genome( genome_words + 4u, 0u );
    typedef PackedStream<uint32*,uint8,2u,true> host_stream;
    host_stream G( &h_genome[0] );
    for (uint32 i = 0; i < genome_len; ++i) G[i] = uint8( rng.below( 4u ) );

    std::vector<int32>  h_sa( genome_len + 1u );
    gen_sa( genome_len, G, &h_sa[0] );
    std::vector<uint32> h_bwt( genome_words + 4u, 0u );
    host_stream B( &h_bwt[0] );
    const uint32 primary = gen_bwt_from_sa( genome_len, G, &h_sa[0], B );
    const uint32 n_blocks = (genome_len + 63u) / 64u;
    std::vector<uint32> h_occ( n_blocks * 4u + 4u, 0u ); uint32 cnt[4];
    build_occurrence_table<2u,64u>( PackedStream<const uint32*,uint8,2u,true>( &h_bwt[0] ), PackedStream<const uint32*,uint8,2u,true>( &h_bwt[0] ) + genome_len, &h_occ[0], cnt );
    std::vector<uint32> h_bwt_occ( n_blocks * 8u );
    for (uint32 k = 0; k < n_blocks; ++k)                              // {uint4 bwt, uint4 occ} per 64 symbols (io/fmindex/fmindex_impl.cu:308-322)
        for (uint32 j = 0; j < 4u; ++j) { h_bwt_occ[ k*8u + j ] = h_bwt[ k*4u + j ]; h_bwt_occ[ k*8u + 4u + j ] = h_occ[ k*4u + j ]; }
    uint32 h_L2[5]; h_L2[0] = 0u; for (uint32 c = 0; c < 4u; ++c) h_L2[c+1] = h_L2[c] + cnt[c];
    const uint32 n_ssa = (genome_len + 16u) / 16u;
    std::vector<uint32> h_ssa( n_ssa );
    {
        SSA_index_multiple<16u> s( genome_len, (const uint32*)&h_sa[0] );
        for (uint32 i = 0; i < n_ssa; ++i) h_ssa[i] = s.m_ssa[i];
        h_ssa[0] = uint32(-1);                                          // io/fmindex/fmindex_impl.cu:244
    }
    uint32 h_ct[256]; gen_bwt_count_table( h_ct );

    const bool dump_inputs = getenv( "SHIM_HARNESS_DUMP_INPUTS" ) != NULL;      // CPU-only debugging aid: write the inputs and stop before any GPU work
    if (dump_inputs)
    {
        dump( out, "in_bwt_occ.bin", h_bwt_occ.data(), h_bwt_occ.size() ); dump( out, "in_ssa.bin", h_ssa.data(), h_ssa.size() );
        uint32 meta[8] = { genome_len, primary, h_L2[0], h_L2[1], h_L2[2], h_L2[3], h_L2[4], 0u };
        dump( out, "in_meta.bin", meta, 8 );
    }
    thrust::device_vector<uint32> d_genome, d_bwt_occ, d_ssa, d_L2, d_ct;
    if (!dump_inputs) { d_genome = h_genome; d_bwt_occ = h_bwt_occ; d_ssa = h_ssa; d_L2.assign( h_L2, h_L2 + 5 ); d_ct.assign( h_ct, h_ct + 256 ); }
    typedef io::FMIndexDataDevice D;
    const D::bwt_occ_type bwt_occ_ptr( (const uint4*)thrust::raw_pointer_cast( d_bwt_occ.data() ) );
    const fm_index_type fm_index(
        genome_len, primary, thrust::raw_pointer_cast( d_L2.data() ),
        D::rank_dict_type( D::bwt_stream_type( D::bwt_type( bwt_occ_ptr ) ), D::occ_type( bwt_occ_ptr ), D::count_table_type( thrust::raw_pointer_cast( d_ct.data() ) ) ),
        D::ssa_type( D::ssa_ldg_type( thrust::raw_pointer_cast( d_ssa.data() ) ) ) );

    // ---- reads: DNA_N, 4 bits per symbol big-endian, string 2r = read r forward, 2r+1 = its reverse complement
    const uint32 n_strings = 2u * n_reads;
    std::vector<uint32> h_index( n_strings + 1u );
    std::vector<uint8>  sym( read_len );
    uint32 total = 0u, max_len = 0u;
    std::vector<uint32> h_reads;
    typedef PackedStream<uint32*,uint8,4u,true> host_read_stream;
    std::vector<uint32> lens( n_reads );
    for (uint32 r = 0; r < n_reads; ++r) { lens[r] = read_len - (r % 7u == 3u ? rng.below( 20u ) : 0u); total += 2u * lens[r]; max_len = nvbio::max( max_len, lens[r] ); }
    h_reads.assign( (total + 7u) / 8u + 4u, 0u );
    host_read_stream R( &h_reads[0] );
    uint32 cursor = 0u;
    for (uint32 r = 0; r < n_reads; ++r)
    {
        const uint32 len = lens[r];
        const uint32 pos = rng.below( genome_len - len - 1u );
        for (uint32 j = 0; j < len; ++j)
        {
            uint8 c = G[pos + j];
            const double u = rng.unit();
            // substitutions only: the reference's match() indexes its tables out of bounds on an N (fmindex_inl.h:329 tests
            // c > symbol_count()), so a seed with an N is undefined behaviour in the reference build
            if (u < 0.02)       c = uint8( (c + 1u + rng.below( 3u )) & 3u );
            sym[j] = c;
        }
        const bool flip = rng.below( 2u ) == 1u;                          // half of the reads come from the reverse strand
        h_index[2u*r] = cursor;
        for (uint32 j = 0; j < len; ++j) { const uint8 c = flip ? (sym[len-1u-j] < 4u ? 3u - sym[len-1u-j] : 4u) : sym[j]; R[cursor + j] = c; }
        cursor += len;
        h_index[2u*r+1u] = cursor;
        for (uint32 j = 0; j < len; ++j) { const uint8 c = R[ h_index[2u*r] + len-1u-j ]; R[cursor + j] = c < 4u ? 3u - c : 4u; }
        cursor += len;
    }
    h_index[n_strings] = cursor;
    if (dump_inputs) { dump( out, "in_reads.bin", h_reads.data(), h_reads.size() ); dump( out, "in_index.bin", h_index.data(), h_index.size() ); return 0; }
    thrust::device_vector<uint32> d_reads( h_reads ), d_index( h_index );

    io::SequenceDataInfo info;
    info.m_alphabet = DNA_N; info.m_n_seqs = n_strings; info.m_name_stream_len = 0u;
    info.m_sequence_stream_len = cursor; info.m_sequence_stream_words = uint32( h_reads.size() );
    info.m_has_qualities = 0u; info.m_min_sequence_len = 1u; info.m_max_sequence_len = max_len; info.m_avg_sequence_len = read_len;
    const io::ConstSequenceDataView reads_view( info, thrust::raw_pointer_cast( d_reads.data() ), thrust::raw_pointer_cast( d_index.data() ), NULL, NULL, NULL );
    const read_access_type reads_access( reads_view );

    std::vector<uint32> h_gindex( 2 ); h_gindex[0] = 0u; h_gindex[1] = genome_len;
    thrust::device_vector<uint32> d_gindex( h_gindex );
    io::SequenceDataInfo ginfo;
    ginfo.m_alphabet = DNA; ginfo.m_n_seqs = 1u; ginfo.m_sequence_stream_len = genome_len; ginfo.m_sequence_stream_words = genome_words;
    ginfo.m_min_sequence_len = ginfo.m_max_sequence_len = ginfo.m_avg_sequence_len = genome_len;
    const io::ConstSequenceDataView genome_view( ginfo, thrust::raw_pointer_cast( d_genome.data() ), thrust::raw_pointer_cast( d_gindex.data() ), NULL, NULL, NULL );
    const genome_access_type genome_access( genome_view );

    // ---- seeds: uniformly spaced infixes of every string, as an InfixSet over the read string-set
    typedef read_access_type::sequence_string_set_type                              read_string_set_type;
    typedef InfixSet<read_string_set_type, const string_set_infix_coord_type*>      seed_string_set_type;
    std::vector<string_set_infix_coord_type> h_seeds;
    for (uint32 s = 0; s < n_strings; ++s)
    {
        const uint32 len = h_index[s+1u] - h_index[s];
        for (uint32 p = 0; p + SEED_LEN <= len; p += SEED_INTV)
            h_seeds.push_back( make_uint4( s, p, p + SEED_LEN, 0u ) );   // (string id, begin, end, -)
    }
    thrust::device_vector<string_set_infix_coord_type> d_seeds( h_seeds );
    const uint32 n_seeds = uint32( h_seeds.size() );
    const read_string_set_type read_string_set = reads_access.sequence_string_set();
    const seed_string_set_type seed_string_set( n_seeds, read_string_set, thrust::raw_pointer_cast( d_seeds.data() ) );

    // ---- rank + locate
    fm_filter_type fm_filter;
    GpuTimer timer; float rank_ms = 1e30f, locate_ms = 1e30f;
    uint64 n_hits = 0u;
    for (int rep = 0; rep < 3; ++rep)
    {
        timer.start();
        n_hits = fm_filter.rank( fm_index, seed_string_set );
        const float ms = timer.stop();
        if (rep && ms < rank_ms) rank_ms = ms;
    }
    cuda_check( "FMIndexFilterDevice::rank" );
    std::vector<uint2>  h_ranges( n_seeds ); std::vector<uint64> h_slots( n_seeds );
    cudaMemcpy( h_ranges.data(), fm_filter.ranges(), sizeof(uint2) * n_seeds, cudaMemcpyDeviceToHost );
    cudaMemcpy( h_slots.data(),  fm_filter.ranks(),  sizeof(uint64) * n_seeds, cudaMemcpyDeviceToHost );
    dump( out, "fmmap_ranges.bin", h_ranges.data(), n_seeds );
    dump( out, "fmmap_slots.bin",  h_slots.data(),  n_seeds );

    const uint32 nh = uint32( n_hits );
    thrust::device_vector<uint2> hits( nh );
    for (int rep = 0; rep < 3; ++rep)
    {
        timer.start();
        // in two batches, to exercise a non-zero `begin`
        const uint64 mid = n_hits / 3u;
        fm_filter.locate( 0u,  mid,    hits.begin() );
        fm_filter.locate( mid, n_hits, hits.begin() + mid );
        const float ms = timer.stop();
        if (rep && ms < locate_ms) locate_ms = ms;
    }
    cuda_check( "FMIndexFilterDevice::locate" );
    dump( out, "fmmap_hits.bin", hits, nh );

    // ---- diagonals, infixes, banded extension, best per read
    const uint32 grid = (nh + 255u) / 256u;
    hits_to_diagonals_kernel<<<grid,256>>>( nh, thrust::raw_pointer_cast( hits.data() ), thrust::raw_pointer_cast( d_seeds.data() ) );
    thrust::device_vector<string_infix_coord_type> read_infix_coords( nh ), genome_infix_coords( nh );
    infixes_kernel<BAND_LEN><<<grid,256>>>( nh, thrust::raw_pointer_cast( hits.data() ), reads_view, genome_len,
                                            thrust::raw_pointer_cast( read_infix_coords.data() ), thrust::raw_pointer_cast( genome_infix_coords.data() ) );
    cuda_check( "infixes" );
    const float ext16_ms = extend_hits<int16>( "i16", out, nh, n_reads, max_len, hits, read_infix_coords, genome_infix_coords, reads_access, genome_access );
    const float ext32_ms = extend_hits<int32>( "i32", out, nh, n_reads, max_len, hits, read_infix_coords, genome_infix_coords, reads_access, genome_access );

    uint64 b200_calls[5] = { 0u, 0u, 0u, 0u, 0u };
#if defined(NVBIO_B200_SHIM)
    { const nvbio::b200::shim_stats& st = nvbio::b200::stats(); b200_calls[0] = st.fm_rank; b200_calls[1] = st.fm_locate; b200_calls[2] = st.banded_score; b200_calls[3] = st.full_score; b200_calls[4] = st.fallbacks; }
#endif
    printf( "{\"program\": \"fmmap\", \"shim\": %d, \"genome_len\": %u, \"reads\": %u, \"seeds\": %u, \"hits\": %llu, \"rank_ms\": %.4f, \"locate_ms\": %.4f, "
            "\"extend_int16_ms\": %.4f, \"extend_int32_ms\": %.4f, \"b200_calls\": {\"fm_rank\": %llu, \"fm_locate\": %llu, \"banded\": %llu, \"full\": %llu, \"fallbacks\": %llu}}\n",
#if defined(NVBIO_B200_SHIM)
            1,
#else
            0,
#endif
            genome_len, n_reads, n_seeds, (unsigned long long)n_hits, rank_ms, locate_ms, ext16_ms, ext32_ms,
            (unsigned long long)b200_calls[0], (unsigned long long)b200_calls[1], (unsigned long long)b200_calls[2], (unsigned long long)b200_calls[3], (unsigned long long)b200_calls[4] );
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// program 2: batch -- a user-defined stream, as an application (or nvbio-test/alignment_test.cu:65-168) would write it
// ---------------------------------------------------------------------------------------------------
namespace nvbio {
namespace aln {

template <typename t_aligner_type, uint32 M, uint32 N>
struct TestStream
{
    typedef t_aligner_type                                                          aligner_type;
    typedef nvbio::cuda::ldg_pointer<uint32>                                        storage_iterator;
    typedef nvbio::lmem_cache_tag<32>                                               cache_type;

    typedef nvbio::PackedStringLoader<storage_iterator,4,false,cache_type>          pattern_loader_type;
    typedef typename pattern_loader_type::input_iterator                            pattern_input;      // PackedStream<ldg,uint8,4,false>
    typedef nvbio::vector_view<typename pattern_loader_type::iterator>              pattern_string;
    typedef nvbio::PackedStringLoader<storage_iterator,2,false,cache_type>          text_loader_type;
    typedef typename text_loader_type::input_iterator                               text_input;         // PackedStream<ldg,uint8,2,false>
    typedef nvbio::vector_view<typename text_loader_type::iterator>                 text_string;

    struct context_type { int32 min_score; aln::BestSink<int32> sink; };
    struct strings_type
    {
        pattern_loader_type     pattern_loader;
        text_loader_type        text_loader;
        pattern_string          pattern;
        trivial_quality_string  quals;
        text_string             text;
    };

    TestStream(aligner_type _aligner, const uint32 _count, const uint32* _patterns, const uint32* _text, int16* _scores,
               const int32 _min_score = Field_traits<int32>::min()) :
        m_aligner( _aligner ), m_count( _count ), m_patterns( storage_iterator( _patterns ) ), m_text( storage_iterator( _text ) ), m_scores( _scores ),
        m_min_score( _min_score ) {}

    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE const aligner_type& aligner() const { return m_aligner; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE uint32 max_pattern_length() const { return M; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE uint32 max_text_length() const { return N; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE uint32 size() const { return m_count; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE uint32 pattern_length(const uint32 i, context_type* context) const { return M; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE uint32 text_length(const uint32 i, context_type* context) const { return N; }

    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE
    bool init_context(const uint32 i, context_type* context) const
    {
        context->min_score = m_min_score;                   // the staged scheduler gives up on alignments that cannot reach it
        context->sink      = aln::BestSink<int32>();
        return (i % 1000u) != 999u;                         // a few alignments are skipped: output() still runs for them
    }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE
    void load_strings(const uint32 i, const uint32 window_begin, const uint32 window_end, const context_type* context, strings_type* strings) const
    {
        strings->pattern = pattern_string( M, strings->pattern_loader.load( m_patterns + i * M, M, make_uint2( window_begin, window_end ), false ) );
        strings->text    = text_string( N, strings->text_loader.load( m_text + i * N, N ) );
    }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE
    void output(const uint32 i, const context_type* context) const
    {
        m_scores[i] = int16( nvbio::max( context->sink.score, int32(-30000) ) );        // the stream's own output rule: a clamp + narrowing
    }

    aligner_type    m_aligner;
    uint32          m_count;
    pattern_input   m_patterns;
    text_input      m_text;
    int16*          m_scores;
    int32           m_min_score;
};

#if defined(NVBIO_B200_SHIM)
// the whole binding of a user stream: where its strings are ...
namespace b200 {
template <typename aligner_type, uint32 M, uint32 N>
struct stream_binding< TestStream<aligner_type,M,N> > : public binding_defaults< TestStream<aligner_type,M,N> >
{
    typedef TestStream<aligner_type,M,N>                            stream_type;
    typedef typename stream_type::context_type                      context_type;
    typedef nvbio::vector_view<typename stream_type::pattern_input> pattern_string;
    typedef nvbio::vector_view<typename stream_type::text_input>    text_string;
    static const bool bound = true;
    static const uint32* pattern_words(const stream_type& s) { return s.m_patterns.stream().m_base; }
    static const uint32* text_words   (const stream_type& s) { return s.m_text.stream().m_base; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static pattern_string pattern(const stream_type& s, const uint32 i, const context_type*) { return pattern_string( M, s.m_patterns + i * M ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static text_string    text   (const stream_type& s, const uint32 i, const context_type*) { return text_string( N, s.m_text + i * N ); }
};
} // namespace b200
// ... and which batch classes forward to the nvbio_b200 kernels
template <uint32 BLOCKDIM, uint32 MINBLOCKS, uint32 BAND_LEN, typename aligner_type, uint32 M, uint32 N>
struct BatchedBandedAlignmentScore< BAND_LEN, TestStream<aligner_type,M,N>, DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > :
    public b200::BandedScoreBatch< BAND_LEN, TestStream<aligner_type,M,N>, DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > {};
template <uint32 BAND_LEN, typename aligner_type, uint32 M, uint32 N>
struct BatchedBandedAlignmentScore< BAND_LEN, TestStream<aligner_type,M,N>, DeviceStagedThreadScheduler > :
    public b200::BandedScoreBatch< BAND_LEN, TestStream<aligner_type,M,N>, DeviceStagedThreadScheduler > {};
#endif

} // namespace aln
} // namespace nvbio

template <uint32 BITS>
static void fill_words(Rng& rng, const uint32 alphabet, const uint64 n_symbols, std::vector<uint32>& words)
{
    typedef PackedStream<uint32*,uint8,BITS,false> stream_t;
    words.assign( (n_symbols * BITS + 31u) / 32u + 4u, 0u );
    stream_t s( &words[0] );
    for (uint64 i = 0; i < n_symbols; ++i) s[i] = uint8( rng.below( alphabet ) );
}

template <uint32 BAND_LEN, uint32 M, uint32 N, typename scheduler_type, typename aligner_type>
static float run_banded_batch(const std::string& out, const char* name, const aligner_type aligner, const uint32 n_tasks,
                              const thrust::device_vector<uint32>& pat, const thrust::device_vector<uint32>& txt,
                              const int32 min_score = Field_traits<int32>::min())
{
    typedef aln::TestStream<aligner_type,M,N>                                       stream_type;
    typedef aln::BatchedBandedAlignmentScore<BAND_LEN,stream_type,scheduler_type>   batch_type;
    thrust::device_vector<int16> scores( n_tasks, int16(-7) );
    stream_type stream( aligner, n_tasks, thrust::raw_pointer_cast( pat.data() ), thrust::raw_pointer_cast( txt.data() ), thrust::raw_pointer_cast( scores.data() ), min_score );
    batch_type batch;
    const uint64 temp_size = batch_type::max_temp_storage( M, N, n_tasks );
    thrust::device_vector<uint8> temp( temp_size ? temp_size : 1u );
    GpuTimer timer; float best_ms = 1e30f;
    for (int rep = 0; rep < 3; ++rep)
    {
        timer.start();
        batch.enact( stream, temp_size, temp_size ? thrust::raw_pointer_cast( temp.data() ) : NULL );
        const float ms = timer.stop();
        if (rep && ms < best_ms) best_ms = ms;
    }
    cuda_check( name );
    dump( out, (std::string("batch_") + name + ".bin").c_str(), scores, n_tasks );
    return best_ms;
}

static int run_batch(const std::string& out, const uint32 n_tasks)
{
    static const uint32 M = 150u;
    Rng rng( 0xD1B54A32D192ED03ull );
    std::string json = "{\"program\": \"batch\", \"n_tasks\": " + std::to_string( n_tasks );
    // texts: random 2-bit; patterns: the text's first M symbols shifted by a small offset with a few edits, so that scores are not trivial
    {
        static const uint32 BAND_LEN = 15u, N = M + BAND_LEN;
        std::vector<uint32> h_txt, h_pat;
        fill_words<2u>( rng, 4u, uint64(N) * n_tasks, h_txt );
        h_pat.assign( (uint64(M) * n_tasks * 4u + 31u) / 32u + 4u, 0u );
        PackedStream<uint32*,uint8,2u,false> T( &h_txt[0] ); PackedStream<uint32*,uint8,4u,false> P( &h_pat[0] );
        for (uint32 t = 0; t < n_tasks; ++t)
        {
            const uint32 shift = rng.below( BAND_LEN / 2u );
            for (uint32 j = 0; j < M; ++j)
            {
                uint8 c = T[ uint64(t) * N + nvbio::min( j + shift, N - 1u ) ];
                const double u = rng.unit();
                if (u < 0.03) c = uint8( rng.below( 4u ) ); else if (u < 0.035) c = 4u;
                P[ uint64(t) * M + j ] = c;
            }
        }
        thrust::device_vector<uint32> pat( h_pat ), txt( h_txt );
        aln::SimpleGotohScheme scoring( 2, -1, -1, -1 );                // nvbio-test/alignment_test.cu:1035-1039
        char buf[256];
        float ms;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceThreadScheduler>( out, "b15_global_thread", aln::make_gotoh_aligner<aln::GLOBAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b15_global_thread_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceThreadScheduler>( out, "b15_semi_thread", aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b15_semi_thread_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceThreadScheduler>( out, "b15_local_thread", aln::make_gotoh_aligner<aln::LOCAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b15_local_thread_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceStagedThreadScheduler>( out, "b15_local_staged", aln::make_gotoh_aligner<aln::LOCAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b15_local_staged_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceStagedThreadScheduler>( out, "b15_global_staged", aln::make_gotoh_aligner<aln::GLOBAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b15_global_staged_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
    }
    {
        static const uint32 BAND_LEN = 31u, N = M + BAND_LEN;
        std::vector<uint32> h_txt, h_pat;
        fill_words<2u>( rng, 4u, uint64(N) * n_tasks, h_txt );
        h_pat.assign( (uint64(M) * n_tasks * 4u + 31u) / 32u + 4u, 0u );
        PackedStream<uint32*,uint8,2u,false> T( &h_txt[0] ); PackedStream<uint32*,uint8,4u,false> P( &h_pat[0] );
        for (uint32 t = 0; t < n_tasks; ++t)
        {
            const uint32 shift = rng.below( BAND_LEN / 2u );
            for (uint32 j = 0; j < M; ++j)
            {
                uint8 c = T[ uint64(t) * N + nvbio::min( j + shift, N - 1u ) ];
                if (rng.unit() < 0.03) c = uint8( rng.below( 4u ) );
                P[ uint64(t) * M + j ] = c;
            }
        }
        thrust::device_vector<uint32> pat( h_pat ), txt( h_txt );
        aln::SimpleGotohScheme scoring( 2, -2, -5, -3 );
        char buf[256];
        float ms;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceThreadScheduler>( out, "b31_local_thread", aln::make_gotoh_aligner<aln::LOCAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b31_local_thread_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
        ms = run_banded_batch<BAND_LEN,M,N,aln::DeviceThreadScheduler>( out, "b31_semi_thread", aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( scoring ), n_tasks, pat, txt );
        snprintf( buf, sizeof(buf), ", \"b31_semi_thread_gcups\": %.2f", 1.0e-6 * double(n_tasks) * BAND_LEN * M / ms ); json += buf;
    }
    // full-matrix DP through the convenience function over packed string sets (what sw-benchmark runs, sw-benchmark.cu:592-641)
    {
        static const uint32 FM = 100u, FN = 400u;
        const uint32 n_full = nvbio::max( n_tasks / 8u, 1024u );
        std::vector<uint32> h_txt, h_pat;
        fill_words<2u>( rng, 4u, uint64(FN) * n_full, h_txt );
        h_pat.assign( (uint64(FM) * n_full * 2u + 31u) / 32u + 4u, 0u );
        PackedStream<uint32*,uint8,2u,false> T( &h_txt[0] ); PackedStream<uint32*,uint8,2u,false> P( &h_pat[0] );
        for (uint32 t = 0; t < n_full; ++t)
        {
            const uint32 shift = rng.below( FN - FM );
            for (uint32 j = 0; j < FM; ++j)
            {
                uint8 c = T[ uint64(t) * FN + j + shift ];
                if (rng.unit() < 0.04) c = uint8( rng.below( 4u ) );
                P[ uint64(t) * FM + j ] = c;
            }
        }
        thrust::device_vector<uint32> pat( h_pat ), txt( h_txt );
        std::vector<uint32> h_poff( n_full + 1u ), h_toff( n_full + 1u );
        for (uint32 t = 0; t <= n_full; ++t) { h_poff[t] = t * FM; h_toff[t] = t * FN; }
        thrust::device_vector<uint32> poff( h_poff ), toff( h_toff );
        typedef PackedStream<const uint32*,uint8,2u,false>          stream_t;
        typedef ConcatenatedStringSet<stream_t,const uint32*>       set_t;
        const set_t patterns( n_full, stream_t( thrust::raw_pointer_cast( pat.data() ) ), thrust::raw_pointer_cast( poff.data() ) );
        const set_t texts   ( n_full, stream_t( thrust::raw_pointer_cast( txt.data() ) ), thrust::raw_pointer_cast( toff.data() ) );
        thrust::device_vector< aln::BestSink<int32> > sinks( n_full );
        const aln::SimpleGotohScheme scoring( 2, -1, -2, -1 );          // sw-benchmark.cu:594-598
        const char* names[3] = { "full_global", "full_local", "full_semi" };
        for (int ty = 0; ty < 3; ++ty)
        {
            GpuTimer timer; float best_ms = 1e30f;
            for (int rep = 0; rep < 3; ++rep)
            {
                timer.start();
                if (ty == 0) aln::batch_alignment_score( aln::make_gotoh_aligner<aln::GLOBAL>( scoring ),      patterns, texts, thrust::raw_pointer_cast( sinks.data() ), aln::DeviceThreadScheduler(), FM, FN );
                if (ty == 1) aln::batch_alignment_score( aln::make_gotoh_aligner<aln::LOCAL>( scoring ),       patterns, texts, thrust::raw_pointer_cast( sinks.data() ), aln::DeviceThreadScheduler(), FM, FN );
                if (ty == 2) aln::batch_alignment_score( aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( scoring ), patterns, texts, thrust::raw_pointer_cast( sinks.data() ), aln::DeviceThreadScheduler(), FM, FN );
                const float ms = timer.stop();
                if (rep && ms < best_ms) best_ms = ms;
            }
            cuda_check( names[ty] );
            thrust::device_vector<int32> score( n_full ); thrust::device_vector<uint2> sink( n_full );
            split_sinks_kernel<<<(n_full + 255u) / 256u,256>>>( n_full, thrust::raw_pointer_cast( sinks.data() ), thrust::raw_pointer_cast( score.data() ), thrust::raw_pointer_cast( sink.data() ) );
            cuda_check( "split" );
            dump( out, (std::string("batch_") + names[ty] + "_scores.bin").c_str(), score, n_full );
            dump( out, (std::string("batch_") + names[ty] + "_sinks.bin").c_str(), sink, n_full );
            char buf[256];
            snprintf( buf, sizeof(buf), ", \"%s_gcups\": %.2f", names[ty], 1.0e-6 * double(n_full) * FM * FN / best_ms ); json += buf;
        }
    }
    uint64 b200_calls[3] = { 0u, 0u, 0u };
#if defined(NVBIO_B200_SHIM)
    { const nvbio::b200::shim_stats& st = nvbio::b200::stats(); b200_calls[0] = st.banded_score; b200_calls[1] = st.full_score; b200_calls[2] = st.fallbacks; }
    json += ", \"shim\": 1";
#else
    json += ", \"shim\": 0";
#endif
    json += ", \"b200_calls\": {\"banded\": " + std::to_string( b200_calls[0] ) + ", \"full\": " + std::to_string( b200_calls[1] ) + ", \"fallbacks\": " + std::to_string( b200_calls[2] ) + "}}";
    printf( "%s\n", json.c_str() );
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// program 3: edges -- the same entry points at the shapes where a forwarding layer goes wrong
// ---------------------------------------------------------------------------------------------------
// One batch of n alignments against windows of a 2-bit big-endian "genome" (a SparseStringSet of (begin, end) ranges), patterns in a
// ConcatenatedStringSet.  Per alignment i, a pattern length L (0, 1..40, 60..200, or 700..830: past 801 - BAND_LEN, the longest
// pattern the packed 16-bit kernels take, so one call mixes both routes) and a window kind:
//   FULL   L + BAND_LEN - 1 symbols            SHORT1  one symbol fewer           RANDOM  a length in [max(L, 62), L + BAND_LEN - 1]
//   BELOW  L - 1 symbols (the DP does not run: the sink keeps its defaults)        EMPTY   no symbols
// and L = 0 (an empty pattern) against a window of 62..67 symbols.
// Why no other windows: the reference's banded kernel loads the first BAND_LEN - 1 text symbols before it looks at the text's
// length (gotoh_banded_inl.h:441-442) and reads past a window of fewer than BAND_LEN - 1 symbols that is not shorter than the
// pattern, so such a window has no defined result.  Every window here that the DP runs on (text_len >= L) has text_len >= BAND_LEN - 1:
// for L >= 1, FULL and SHORT1 have L + BAND_LEN - 1 and L + BAND_LEN - 2 >= BAND_LEN - 1 symbols and RANDOM at least 62 >= BAND_LEN - 1;
// an empty pattern gets 62..67.
// The staged scheduler loads BAND_LEN - 1 symbols from every 32-row window's start (batched_stream.h:161-176), so its batch uses
// FULL in place of RANDOM (every other kind keeps that load inside the window).
enum { W_FULL = 0, W_SHORT1, W_RANDOM, W_BELOW, W_EMPTY, W_KINDS };
static const uint32 EDGE_MAX_P = 830u, EDGE_MIN_T = 62u, EDGE_MAX_BAND = 63u;

struct EdgeInputs
{
    uint32 n;
    std::vector<uint32> genome;                  // 2-bit big-endian words
    std::vector<uint32> p_len, p_sym_off;        // pattern i: symbols [p_sym_off, +p_len) of the pattern stream
    std::vector<uint8>  p_sym;                   // 0..3, 4 = N
    std::vector<uint32> t_begin, kind;           // window i begins at t_begin[i]; its length depends on the band and the kind
    uint32 genome_len;
};

static EdgeInputs make_edge_inputs(Rng& rng, const uint32 n)
{
    EdgeInputs in; in.n = n;
    in.genome_len = n * 40u + 4096u;
    in.genome.assign( in.genome_len / 16u + 8u, 0u );
    PackedStream<uint32*,uint8,2u,true> G( &in.genome[0] );
    for (uint32 i = 0; i < in.genome_len; ++i) G[i] = uint8( rng.below( 4u ) );
    uint32 off = 0u;
    for (uint32 i = 0; i < n; ++i)
    {
        const uint32 c = rng.below( 100u );
        const uint32 L = c < 3u ? 0u : c < 20u ? 1u + rng.below( 40u ) : c < 90u ? 60u + rng.below( 141u ) : 700u + rng.below( EDGE_MAX_P - 700u + 1u );
        const uint32 k = L == 0u ? W_RANDOM : (i % 11u == 3u ? W_BELOW : i % 11u == 7u ? W_EMPTY : i % 5u == 1u ? W_SHORT1 : i % 5u == 2u ? W_RANDOM : W_FULL);
        const uint32 begin = rng.below( in.genome_len - EDGE_MAX_P - EDGE_MAX_BAND - 8u );
        in.p_len.push_back( L ); in.p_sym_off.push_back( off ); in.t_begin.push_back( begin ); in.kind.push_back( k );
        // the pattern: the window's text shifted by a few symbols, with substitutions, N's (1 in 8 patterns) and the odd deletion
        const uint32 shift = rng.below( 4u );
        const bool with_n = rng.below( 8u ) == 0u;
        uint32 src = begin + shift;
        for (uint32 j = 0; j < L; ++j)
        {
            if (rng.below( 200u ) == 0u) src += 1u + rng.below( 2u );
            uint8 s = uint8( G[src++] );
            const double u = rng.unit();
            if (u < 0.03) s = uint8( (s + 1u + rng.below( 3u )) & 3u );
            else if (with_n && u < 0.05) s = 4u;
            in.p_sym.push_back( s );
        }
        off += L;
    }
    return in;
}

static uint32 edge_window_len(const EdgeInputs& in, const uint32 i, const uint32 band, const bool staged, Rng& rng)
{
    const uint32 L = in.p_len[i];
    if (L == 0u) return EDGE_MIN_T + rng.below( 6u );
    switch (in.kind[i])
    {
    case W_SHORT1: return L + band - 2u;
    case W_BELOW:  return L - 1u;
    case W_EMPTY:  return 0u;
    case W_RANDOM: if (!staged) { const uint32 lo = nvbio::max( L, EDGE_MIN_T ), hi = L + band - 1u; return lo >= hi ? hi : lo + rng.below( hi - lo + 1u ); }
    default:       return L + band - 1u;
    }
}

/// the pattern symbols packed BITS per symbol (2-bit patterns: an N becomes A, as a 2-bit packer would store it)
template <uint32 BITS, bool BE>
static std::vector<uint32> pack_patterns(const EdgeInputs& in)
{
    std::vector<uint32> w( (in.p_sym.size() * BITS + 31u) / 32u + 8u, 0u );
    PackedStream<uint32*,uint8,BITS,BE> P( &w[0] );
    for (size_t j = 0; j < in.p_sym.size(); ++j) P[j] = BITS == 2u ? uint8( in.p_sym[j] & 3u ) : in.p_sym[j];
    return w;
}

struct EdgeRun
{
    std::string out, json;
    uint32 banded_calls, full_calls, fallback_calls;
    EdgeRun(const std::string& o) : out( o ), banded_calls( 0u ), full_calls( 0u ), fallback_calls( 0u ) {}
    void add(const std::string& key, const uint64 v) { json += ", \"" + key + "\": " + std::to_string( v ); }
};

template <typename sink_type>
static void dump_sinks(EdgeRun& run, const std::string& name, const thrust::device_vector<sink_type>& sinks, const uint32 n)
{
    thrust::device_vector<int32> score( n ); thrust::device_vector<uint2> sink( n );
    if (n) split_sinks_kernel<<<(n + 255u) / 256u,256>>>( n, thrust::raw_pointer_cast( sinks.data() ), thrust::raw_pointer_cast( score.data() ), thrust::raw_pointer_cast( sink.data() ) );
    cuda_check( name.c_str() );
    dump( run.out, (name + "_scores.bin").c_str(), score, n );
    dump( run.out, (name + "_sinks.bin").c_str(), sink, n );
}

/// one aln::batch_banded_alignment_score<BAND_LEN> call over the edge inputs (the first n alignments), through priv::AlignmentStream
template <uint32 BAND_LEN, typename sink_score, uint32 PBITS, bool PBE, typename aligner_type, typename scheduler_type>
static void edge_banded(EdgeRun& run, const std::string& name, const EdgeInputs& in, const uint32 n, const aligner_type aligner,
                        const scheduler_type scheduler, const bool staged, const bool fallback = false)
{
    typedef PackedStream<const uint32*,uint8,PBITS,PBE>                 pattern_stream;
    typedef PackedStream<const uint32*,uint8,2u,true>                   text_stream;
    typedef ConcatenatedStringSet<pattern_stream,const uint32*>         pattern_set;
    typedef SparseStringSet<text_stream,const uint2*>                   text_set;
    Rng rng( 0x5851F42D4C957F2Dull + BAND_LEN );                        // window lengths: the same for every call with this band
    std::vector<uint32> poff( n + 1u ); std::vector<uint2> trange( n );
    uint32 max_p = 1u, max_t = 1u;
    for (uint32 i = 0; i < n; ++i)
    {
        const uint32 tl = edge_window_len( in, i, BAND_LEN, staged, rng );
        poff[i] = in.p_sym_off[i]; trange[i] = make_uint2( in.t_begin[i], in.t_begin[i] + tl );
        max_p = nvbio::max( max_p, in.p_len[i] ); max_t = nvbio::max( max_t, tl );
    }
    poff[n] = n ? in.p_sym_off[n-1u] + in.p_len[n-1u] : 0u;
    const std::vector<uint32> h_pat = pack_patterns<PBITS,PBE>( in );
    thrust::device_vector<uint32> d_pat( h_pat ), d_txt( in.genome ), d_poff( poff );
    thrust::device_vector<uint2>  d_trange( trange );
    const pattern_set patterns( n, pattern_stream( thrust::raw_pointer_cast( d_pat.data() ) ), thrust::raw_pointer_cast( d_poff.data() ) );
    const text_set    texts( n, text_stream( thrust::raw_pointer_cast( d_txt.data() ) ), thrust::raw_pointer_cast( d_trange.data() ) );
    thrust::device_vector< aln::BestSink<sink_score> > sinks( nvbio::max( n, 1u ) );
    aln::batch_banded_alignment_score<BAND_LEN>( aligner, patterns, texts, thrust::raw_pointer_cast( sinks.data() ), scheduler, max_p, max_t );
    dump_sinks( run, name, sinks, n );
    if (fallback) run.fallback_calls++; else run.banded_calls++;
}

/// the same on the harness's user-bound TestStream (fixed M x (M + BAND_LEN) strings, 4-bit little-endian patterns)
template <uint32 BAND_LEN, typename scheduler_type, typename aligner_type>
static void edge_test_stream(EdgeRun& run, const char* name, Rng& rng, const uint32 n, const aligner_type aligner, const bool fallback = false,
                             const int32 min_score = Field_traits<int32>::min())
{
    static const uint32 M = 150u, N = M + BAND_LEN;
    std::vector<uint32> h_txt, h_pat;
    fill_words<2u>( rng, 4u, uint64(N) * n, h_txt );
    h_pat.assign( (uint64(M) * n * 4u + 31u) / 32u + 4u, 0u );
    PackedStream<uint32*,uint8,2u,false> T( &h_txt[0] ); PackedStream<uint32*,uint8,4u,false> P( &h_pat[0] );
    for (uint32 t = 0; t < n; ++t)
    {
        const uint32 shift = rng.below( BAND_LEN / 2u + 1u );
        for (uint32 j = 0; j < M; ++j)
        {
            uint8 c = T[ uint64(t) * N + nvbio::min( j + shift, N - 1u ) ];
            const double u = rng.unit();
            if (u < 0.03) c = uint8( rng.below( 4u ) ); else if (u < 0.035) c = 4u;
            P[ uint64(t) * M + j ] = c;
        }
    }
    thrust::device_vector<uint32> pat( h_pat ), txt( h_txt );
    run_banded_batch<BAND_LEN,M,N,scheduler_type>( run.out, name, aligner, n, pat, txt, min_score );
    if (fallback) run.fallback_calls += 3u; else run.banded_calls += 3u;     // run_banded_batch enacts three times
}

/// full matrix through aln::batch_alignment_score: mixed (M, N) in one batch, some N < M
template <typename sink_score, typename aligner_type>
static void edge_full(EdgeRun& run, const std::string& name, const EdgeInputs& in, const uint32 n, const aligner_type aligner)
{
    typedef PackedStream<const uint32*,uint8,4u,false>                  pattern_stream;
    typedef PackedStream<const uint32*,uint8,2u,true>                   text_stream;
    typedef ConcatenatedStringSet<pattern_stream,const uint32*>         pattern_set;
    typedef SparseStringSet<text_stream,const uint2*>                   text_set;
    Rng rng( 0x1B873593ull );
    // patterns: the first n non-empty patterns of the edge inputs cut to at most 300 symbols; texts of 1..600 symbols, a fifth of them
    // shorter than their pattern (the full-matrix DP takes every pattern and text length >= 1)
    std::vector<uint32> poff; std::vector<uint2> trange;
    uint32 max_p = 1u, max_t = 1u;
    for (uint32 i = 0; poff.size() < n && i < in.n; ++i)
    {
        if (in.p_len[i] == 0u) continue;
        const uint32 L = nvbio::min( in.p_len[i], 300u );
        const uint32 tl = rng.below( 5u ) == 0u ? 1u + rng.below( L ) : L + rng.below( 301u );
        poff.push_back( in.p_sym_off[i] ); trange.push_back( make_uint2( in.t_begin[i], in.t_begin[i] + tl ) );
        max_p = nvbio::max( max_p, L ); max_t = nvbio::max( max_t, tl );
    }
    const uint32 m = uint32( poff.size() );
    // a ConcatenatedStringSet takes lengths from consecutive offsets: give each pattern its own copy of L symbols instead
    std::vector<uint8> sym; std::vector<uint32> off( m + 1u );
    {
        uint32 t = 0u;
        for (uint32 i = 0; t < m && i < in.n; ++i)
        {
            if (in.p_len[i] == 0u) continue;
            const uint32 L = nvbio::min( in.p_len[i], 300u );
            off[t++] = uint32( sym.size() );
            for (uint32 j = 0; j < L; ++j) sym.push_back( in.p_sym[ in.p_sym_off[i] + j ] );
        }
        off[m] = uint32( sym.size() );
    }
    std::vector<uint32> h_pat( (sym.size() * 4u + 31u) / 32u + 8u, 0u );
    { PackedStream<uint32*,uint8,4u,false> P( &h_pat[0] ); for (size_t j = 0; j < sym.size(); ++j) P[j] = sym[j]; }
    thrust::device_vector<uint32> d_pat( h_pat ), d_txt( in.genome ), d_poff( off );
    thrust::device_vector<uint2>  d_trange( trange );
    const pattern_set patterns( m, pattern_stream( thrust::raw_pointer_cast( d_pat.data() ) ), thrust::raw_pointer_cast( d_poff.data() ) );
    const text_set    texts( m, text_stream( thrust::raw_pointer_cast( d_txt.data() ) ), thrust::raw_pointer_cast( d_trange.data() ) );
    thrust::device_vector< aln::BestSink<sink_score> > sinks( m );
    aln::batch_alignment_score( aligner, patterns, texts, thrust::raw_pointer_cast( sinks.data() ), aln::DeviceThreadScheduler(), max_p, max_t );
    dump_sinks( run, name, sinks, m );
    run.full_calls++;
}

static int run_edges(const std::string& out, const uint32 n)
{
    Rng rng( 0xA0761D6478BD642Full );
    const EdgeInputs in = make_edge_inputs( rng, n );
    EdgeRun run( out );
    run.json = "{\"program\": \"edges\", \"n\": " + std::to_string( n );
    // what the batch holds: pattern lengths per route, window kinds, N's
    {
        uint64 empty_p = 0u, long_p = 0u, with_n = 0u, kinds[W_KINDS] = { 0u, 0u, 0u, 0u, 0u };
        for (uint32 i = 0; i < n; ++i)
        {
            if (in.p_len[i] == 0u) ++empty_p; else kinds[ in.kind[i] ]++;
            if (in.p_len[i] > 801u - EDGE_MAX_BAND) ++long_p;
            for (uint32 j = 0; j < in.p_len[i]; ++j) if (in.p_sym[ in.p_sym_off[i] + j ] == 4u) { ++with_n; break; }
        }
        run.add( "empty_patterns", empty_p ); run.add( "long_patterns", long_p ); run.add( "patterns_with_n", with_n );
        run.add( "full_windows", kinds[W_FULL] ); run.add( "short1_windows", kinds[W_SHORT1] ); run.add( "random_windows", kinds[W_RANDOM] );
        run.add( "below_windows", kinds[W_BELOW] ); run.add( "empty_windows", kinds[W_EMPTY] );
    }
    const aln::SimpleGotohScheme sc( 2, -2, -5, -3 );
    const aln::DeviceThreadScheduler thread;
    const aln::DeviceStagedThreadScheduler staged;

    // every band the shim accelerates x the three alignment types, BestSink<int32>, 4-bit little-endian patterns with N's
#define EDGE_TYPES(B) \
    edge_banded<B,int32,4u,false>( run, "b" #B "_global", in, n, aln::make_gotoh_aligner<aln::GLOBAL>( sc ), thread, false ); \
    edge_banded<B,int32,4u,false>( run, "b" #B "_local",  in, n, aln::make_gotoh_aligner<aln::LOCAL>( sc ), thread, false ); \
    edge_banded<B,int32,4u,false>( run, "b" #B "_semi",   in, n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( sc ), thread, false ); \
    edge_banded<B,int16,4u,false>( run, "b" #B "_local_i16", in, n, aln::make_gotoh_aligner<aln::LOCAL>( sc ), thread, false );
    EDGE_TYPES(3) EDGE_TYPES(5) EDGE_TYPES(7) EDGE_TYPES(15) EDGE_TYPES(31) EDGE_TYPES(63)
#undef EDGE_TYPES
    edge_banded<15,int16,4u,false>( run, "b15_global_i16", in, n, aln::make_gotoh_aligner<aln::GLOBAL>( sc ), thread, false );
    edge_banded<15,int16,4u,false>( run, "b15_semi_i16",   in, n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( sc ), thread, false );
    // the other packings: 4-bit big-endian, 2-bit big- and little-endian patterns
    edge_banded<31,int32,4u,true >( run, "b31_local_p4be",  in, n, aln::make_gotoh_aligner<aln::LOCAL>( sc ), thread, false );
    edge_banded<31,int32,2u,true >( run, "b31_global_p2be", in, n, aln::make_gotoh_aligner<aln::GLOBAL>( sc ), thread, false );
    edge_banded<31,int32,2u,false>( run, "b31_semi_p2le",   in, n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( sc ), thread, false );
    // the staged scheduler over priv::AlignmentStream
    edge_banded<15,int32,4u,false>( run, "b15_global_staged", in, n, aln::make_gotoh_aligner<aln::GLOBAL>( sc ), staged, true );
    edge_banded<63,int32,4u,false>( run, "b63_local_staged",  in, n, aln::make_gotoh_aligner<aln::LOCAL>( sc ), staged, true );
    edge_banded<3,int16,4u,false> ( run, "b3_semi_staged_i16", in, n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( sc ), staged, true );
    // deliberate fall-backs: a band the kernels do not implement runs the reference's own kernel
    edge_banded<9,int32,4u,false>( run, "b9_local_fallback", in, n, aln::make_gotoh_aligner<aln::LOCAL>( sc ), thread, false, true );
    // scratch arenas: grow, reuse at the boundaries of the layout kernels' 128-thread blocks, grow again, shrink
    {
        const uint32 sizes[6] = { 1u, 127u, 128u, 129u, n, 5u };
        for (uint32 s = 0; s < 6u; ++s)
            edge_banded<31,int32,4u,false>( run, "b31_global_n" + std::to_string( sizes[s] ) + "_" + std::to_string( s ), in, sizes[s], aln::make_gotoh_aligner<aln::GLOBAL>( sc ), thread, false );
    }
    // scores outside the int16 range: 150 bp near-exact patterns under (300, -200, -500, -300)
    {
        Rng r2( 0x9FB21C651E98DF25ull );
        EdgeInputs big = make_edge_inputs( r2, 2048u );
        for (uint32 i = 0; i < big.n; ++i) { big.kind[i] = W_FULL; }
        // cut every pattern to 150 symbols (or keep it shorter) by rebuilding the pattern stream
        std::vector<uint8> sym; std::vector<uint32> len, off;
        for (uint32 i = 0; i < big.n; ++i)
        {
            const uint32 L = big.p_len[i] == 0u ? 0u : 150u;
            off.push_back( uint32( sym.size() ) ); len.push_back( L );
            PackedStream<const uint32*,uint8,2u,true> G( &big.genome[0] );
            for (uint32 j = 0; j < L; ++j) { uint8 c = uint8( G[ big.t_begin[i] + 3u + j ] ); if (r2.below( 100u ) == 0u) c = uint8( (c + 1u) & 3u ); sym.push_back( c ); }
        }
        big.p_sym = sym; big.p_len = len; big.p_sym_off = off;
        const aln::SimpleGotohScheme wide( 300, -200, -500, -300 );
        edge_banded<15,int32,4u,false>( run, "wide_b15_global",     big, big.n, aln::make_gotoh_aligner<aln::GLOBAL>( wide ), thread, false );
        edge_banded<15,int32,4u,false>( run, "wide_b15_local",      big, big.n, aln::make_gotoh_aligner<aln::LOCAL>( wide ), thread, false );
        edge_banded<15,int32,4u,false>( run, "wide_b15_semi",       big, big.n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( wide ), thread, false );
        edge_banded<15,int16,4u,false>( run, "wide_b15_global_i16", big, big.n, aln::make_gotoh_aligner<aln::GLOBAL>( wide ), thread, false );
        // BestSink<int16>: GLOBAL reports once and stays accelerated; LOCAL and SEMI_GLOBAL keep the best of many narrowed reports, which
        // one report of the int32 best cannot reproduce once scores leave the int16 range, so the shim runs the reference's kernel
        edge_banded<15,int16,4u,false>( run, "wide_b15_local_i16",  big, big.n, aln::make_gotoh_aligner<aln::LOCAL>( wide ), thread, false, true );
        edge_banded<15,int16,4u,false>( run, "wide_b15_semi_i16",   big, big.n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( wide ), thread, false, true );
        // the staged scheduler carries the band between 32-row windows in short2 checkpoints: H near 37,000 at row 128 wraps there, so
        // the reference's staged scores differ from one pass and the shim runs the reference's staged kernel
        edge_banded<15,int32,4u,false>( run, "wide_b15_global_staged", big, big.n, aln::make_gotoh_aligner<aln::GLOBAL>( wide ), staged, true, true );
        edge_banded<15,int32,4u,false>( run, "wide_b15_local_staged",  big, big.n, aln::make_gotoh_aligner<aln::LOCAL>( wide ), staged, true, true );
        edge_banded<15,int32,4u,false>( run, "wide_b15_semi_staged",   big, big.n, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( wide ), staged, true, true );
    }
    // the user-bound stream at the outer bands, both schedulers, and one band it does not take
    {
        Rng r3( 0xE7037ED1A0B428DBull );
        const uint32 nt = 4096u;
        edge_test_stream<3, aln::DeviceThreadScheduler>      ( run, "ts_b3_global_thread", r3, nt, aln::make_gotoh_aligner<aln::GLOBAL>( sc ) );
        edge_test_stream<63,aln::DeviceStagedThreadScheduler>( run, "ts_b63_semi_staged",  r3, nt, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( sc ) );
        edge_test_stream<5, aln::DeviceStagedThreadScheduler>( run, "ts_b5_local_staged",  r3, nt, aln::make_gotoh_aligner<aln::LOCAL>( sc ) );
        edge_test_stream<9, aln::DeviceThreadScheduler>      ( run, "ts_b9_local_fallback", r3, nt, aln::make_gotoh_aligner<aln::LOCAL>( sc ), true );
        // a min_score in reach (150 bp x match 2 = 300 at most): the staged scheduler gives up on alignments that fall behind after a
        // 32-row window, so the shim runs the reference's staged kernel; under the thread scheduler min_score changes nothing
        edge_test_stream<15,aln::DeviceStagedThreadScheduler>( run, "ts_b15_local_staged_min", r3, nt, aln::make_gotoh_aligner<aln::LOCAL>( sc ), true, 200 );
        edge_test_stream<15,aln::DeviceThreadScheduler>      ( run, "ts_b15_local_thread_min", r3, nt, aln::make_gotoh_aligner<aln::LOCAL>( sc ), false, 200 );
    }
    // full matrix
    {
        const uint32 nf = nvbio::min( n, 3000u );
        const aln::SimpleGotohScheme fs( 2, -1, -2, -1 );
        edge_full<int32>( run, "full_global",     in, nf, aln::make_gotoh_aligner<aln::GLOBAL>( fs ) );
        edge_full<int32>( run, "full_local",      in, nf, aln::make_gotoh_aligner<aln::LOCAL>( fs ) );
        edge_full<int32>( run, "full_semi",       in, nf, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( fs ) );
        edge_full<int16>( run, "full_global_i16", in, nf, aln::make_gotoh_aligner<aln::GLOBAL>( fs ) );
        edge_full<int16>( run, "full_local_i16",  in, nf, aln::make_gotoh_aligner<aln::LOCAL>( fs ) );
        edge_full<int16>( run, "full_semi_i16",   in, nf, aln::make_gotoh_aligner<aln::SEMI_GLOBAL>( fs ) );
    }
    uint64 b200_calls[3] = { 0u, 0u, 0u };
#if defined(NVBIO_B200_SHIM)
    { const nvbio::b200::shim_stats& st = nvbio::b200::stats(); b200_calls[0] = st.banded_score; b200_calls[1] = st.full_score; b200_calls[2] = st.fallbacks; }
    run.json += ", \"shim\": 1";
#else
    run.json += ", \"shim\": 0";
#endif
    run.json += ", \"planned\": {\"banded\": " + std::to_string( run.banded_calls ) + ", \"full\": " + std::to_string( run.full_calls ) +
                ", \"fallbacks\": " + std::to_string( run.fallback_calls ) + "}";
    run.json += ", \"b200_calls\": {\"banded\": " + std::to_string( b200_calls[0] ) + ", \"full\": " + std::to_string( b200_calls[1] ) + ", \"fallbacks\": " + std::to_string( b200_calls[2] ) + "}}";
    printf( "%s\n", run.json.c_str() );
    return 0;
}

int main(int argc, char** argv)
{
    if (argc < 3) { fprintf( stderr, "usage: shim_harness fmmap|batch|edges <outdir> [sizes...]\n" ); return 1; }
    const std::string mode = argv[1], out = argv[2];
    try
    {
        if (mode == "fmmap")
            return run_fmmap( out, argc > 3 ? uint32( atoll( argv[3] ) ) : 4000000u, argc > 4 ? uint32( atoll( argv[4] ) ) : 50000u, argc > 5 ? uint32( atoll( argv[5] ) ) : 100u );
        if (mode == "batch")
            return run_batch( out, argc > 3 ? uint32( atoll( argv[3] ) ) : 65536u );
        if (mode == "edges")
            return run_edges( out, argc > 3 ? uint32( atoll( argv[3] ) ) : 20000u );
    }
    catch (const std::exception& e) { fprintf( stderr, "exception: %s\n", e.what() ); return 4; }
    return 1;
}
