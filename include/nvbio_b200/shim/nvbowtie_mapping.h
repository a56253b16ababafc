// nvbio_b200/shim/nvbowtie_mapping.h -- nvBowtie's seed-mapping entry points (SURVEY 8b, boundary B-A2) over the nvbio_b200 kernels.
//
// nvBowtie declares its mapping stage as NON-template functions over its own PODs (nvBowtie/bowtie2/cuda/mapping.h):
//     map / map_exact / map_approx (ReadsDef::type, FMIndexDef::type fmi, rfmi, retry, PingPongQueuesView<uint32>, uint8* reseed,
//                                   SeedHitDequeArrayDeviceView hits, ParamsPOD, bool fw, bool rc)          mapping.cu:77-188
// and defines them in mapping.cu as launches of map_queues_kernel<ALGO> (mapping_inl.h:539-591).  A translation unit that does
//     #define NVBIO_B200_DEFINE_NVBOWTIE_MAPPING
//     #include <nvbio_b200/shim/nvbowtie_mapping.h>
// defines the SAME symbols (same signatures, same namespace) and is compiled and linked IN PLACE OF mapping.cu: the rest of
// nvBowtie (aligner_best_approx.h:162,227, aligner_all.h, ...) links against it unchanged.  The queue forms of map_exact /
// map_approx / map go through nvb_map_seeds; the forms the nvbio_b200 kernels do not cover (case pruning, which needs the reverse index;
// the seed_range forms; map_whole_read; gather_ranges) forward to the reference's own templates, at compile time.
//
// What stays with the reference's types: reads, index, queues, params and the hit deques are read and written in nvBowtie's own
// layouts -- each read's deque is allocated with SeedHitDequeArrayDeviceView::alloc_deque and left as a valid interval heap
// (priority_deque over hit_compare), exactly what the select stage expects (seed_hit_deque_array.h:157-204).
#pragma once

#include <nvBowtie/bowtie2/cuda/mapping.h>
#include <nvBowtie/bowtie2/cuda/mapping_inl.h>
#include <nvbio_b200/shim/views.h>

namespace nvbio {
namespace bowtie2 {
namespace cuda {
namespace b200 {

/// per read: its length and nvBowtie's seed interval, evaluated on the device with the reference's own SimpleFunc (float math
/// under the caller's compiler flags, as in map_queues_kernel, mapping_inl.h:563-565)
template <typename BatchType>
__global__ void read_layout_kernel(const BatchType reads, const ParamsPOD params, uint32* offsets, uint32* lengths, uint32* seed_freq)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= reads.size()) return;
    const uint2  range = reads.get_range( i );
    const uint32 len   = range.y - range.x;
    offsets[i] = range.x; lengths[i] = len;
    seed_freq[i] = len ? (uint32)params.seed_freq( len ) : 1u;
}

/// move every queued read's hits (sorted slots of the nvbio_b200 arena) into nvBowtie's deque array
inline __global__ void store_deques_kernel(const nvbio::cuda::PingPongQueuesView<uint32> queues, const uint32* lengths, const uint32 min_read_len,
                                           const uint32 max_hits, const uint2* slots, const uint32* counts, SeedHitDequeArrayDeviceView hits)
{
    const uint32 id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= queues.in_size) return;
    const uint32 read_id = queues.in_queue[id];
    if (lengths[read_id] < min_read_len) { hits.resize_deque( read_id, 0u ); return; }      // mapping_inl.h:547-551
    const uint32 n = counts[read_id];
    SeedHit* dst = hits.alloc_deque( read_id, n );                                          // store_deque, mapping_inl.h:101-115
    if (dst != NULL)
    {
        hits.resize_deque( read_id, n );
        uint2* d = reinterpret_cast<uint2*>( dst );                                          // SeedHit is two 32-bit words (seed_hit.h:230-232)
        for (uint32 i = 0; i < n; ++i) d[i] = slots[ size_t(read_id) * max_hits + i ];
        // leave a valid interval heap behind (the deque is re-opened with build_heap = false later on)
        typedef SeedHitDequeArrayDeviceView::hit_vector_type hit_vector_type;
        typedef SeedHitDequeArrayDeviceView::hit_deque_type  hit_deque_type;
        hit_deque_type heap( hit_vector_type( n, dst ), false );
    }
}

struct map_workspace
{
    thrust::device_vector<uint32> layout;       // offsets | lengths | seed_freq
    thrust::device_vector<uint2>  slots;
    thrust::device_vector<uint32> counts;
};
inline map_workspace& workspace() { static map_workspace w; return w; }

template <typename BatchType, typename FMType>
struct is_supported
{
    typedef typename BatchType::sequence_stream_type stream_type;
    static const bool value = nvbio::b200::fm_index_view<FMType>::supported && nvbio::b200::packed_iterator<stream_type>::supported &&
                              BatchType::SEQUENCE_BIG_ENDIAN;
};

/// map_queues_kernel<EXACT_MAPPING | APPROX_MAPPING> through nvb_map_seeds
template <typename BatchType, typename FMType>
void map_queues(const uint32 algorithm, const BatchType& reads, const FMType fmi, const uint32 retry,
                const nvbio::cuda::PingPongQueuesView<uint32> queues, uint8* reseed, SeedHitDequeArrayDeviceView hits,
                const ParamsPOD params, const bool fw, const bool rc)
{
    const uint32 n_reads = reads.size();
    if (n_reads == 0u || queues.in_size == 0u) return;
    map_workspace& w = workspace();
    w.layout.resize( 3u * size_t(n_reads) );
    w.slots.resize( size_t(n_reads) * params.max_hits );
    w.counts.resize( n_reads );
    uint32* d_off = thrust::raw_pointer_cast( w.layout.data() );
    uint32* d_len = d_off + n_reads; uint32* d_freq = d_len + n_reads;
    read_layout_kernel<<< (n_reads + 127u) / 128u, 128u >>>( reads, params, d_off, d_len, d_freq );

    typedef typename BatchType::sequence_stream_type stream_type;
    nvb_string_set rs;
    rs.d_words = (const uint32_t*)nvbio::b200::packed_iterator<stream_type>::words( reads.sequence_stream() );
    rs.bits = BatchType::SEQUENCE_BITS; rs.big_endian = 1u;
    rs.d_offsets = d_off; rs.d_lengths = d_len; rs.stride = 0u; rs.length = reads.max_sequence_len();
    const nvb_fm_index index = nvbio::b200::fm_index_view<FMType>::get( fmi );
    nvb_map_params p;
    p.algorithm = algorithm; p.seed_len = params.seed_len; p.seed_freq = 0u; p.max_hits = params.max_hits; p.max_reseed = params.max_reseed;
    p.rep_seeds = params.rep_seeds; p.subseed_len = params.subseed_len; p.min_read_len = params.min_read_len; p.fw = fw ? 1u : 0u; p.rc = rc ? 1u : 0u;
    nvbio::b200::check( nvb_map_seeds( &index, &rs, queues.in_queue, queues.in_size, retry, &p, d_freq,
                                       (nvb_seed_hit*)thrust::raw_pointer_cast( w.slots.data() ), thrust::raw_pointer_cast( w.counts.data() ),
                                       reseed, NULL, NULL ), "nvb_map_seeds" );
    store_deques_kernel<<< (queues.in_size + 127u) / 128u, 128u >>>( queues, d_len, params.min_read_len, params.max_hits,
                                                                     thrust::raw_pointer_cast( w.slots.data() ), thrust::raw_pointer_cast( w.counts.data() ), hits );
    nvbio::b200::stats().fm_rank++;
}

} // namespace b200

#if defined(NVBIO_B200_DEFINE_NVBOWTIE_MAPPING)
// ---- the entry points of nvBowtie/bowtie2/cuda/mapping.cu ------------------------------------------------------------------
void map_exact(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi, const uint32 retry,
               const nvbio::cuda::PingPongQueuesView<uint32> queues, uint8* reseed, SeedHitDequeArrayDeviceView hits,
               const ParamsPOD params, const bool fw, const bool rc)
{
    if (b200::is_supported<ReadsDef::type,FMIndexDef::type>::value)
        b200::map_queues( NVB_MAP_EXACT, read_batch, fmi, retry, queues, reseed, hits, params, fw, rc );
    else
    {
        map_exact_t( read_batch, fmi, rfmi, retry, queues, reseed, hits, params, fw, rc );
        nvbio::b200::stats().fallbacks++;
    }
}
void map_approx(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi, const uint32 retry,
                const nvbio::cuda::PingPongQueuesView<uint32> queues, uint8* reseed, SeedHitDequeArrayDeviceView hits,
                const ParamsPOD params, const bool fw, const bool rc)
{
    if (b200::is_supported<ReadsDef::type,FMIndexDef::type>::value && 3u * params.seed_len + 1u <= NVB_MAP_MAX_PUSHES)
        b200::map_queues( NVB_MAP_APPROX, read_batch, fmi, retry, queues, reseed, hits, params, fw, rc );
    else
    {
        map_approx_t( read_batch, fmi, rfmi, retry, queues, reseed, hits, params, fw, rc );
        nvbio::b200::stats().fallbacks++;
    }
}
void map(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi, const uint32 retry,
         const nvbio::cuda::PingPongQueuesView<uint32> queues, uint8* reseed, SeedHitDequeArrayDeviceView hits,
         const ParamsPOD params, const bool fw, const bool rc)
{
    // the dispatch of map_t (mapping_inl.h:816-855)
    if (params.allow_sub)
    {
        if (params.subseed_len == 0) { map_case_pruning_t( read_batch, fmi, rfmi, retry, queues, reseed, hits, params, fw, rc ); nvbio::b200::stats().fallbacks++; }   // needs the reverse index: reference
        else                         map_approx( read_batch, fmi, rfmi, retry, queues, reseed, hits, params, fw, rc );
    }
    else
        map_exact( read_batch, fmi, rfmi, retry, queues, reseed, hits, params, fw, rc );
}
// forms that stay on the reference's templates
void map_exact(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi, SeedHitDequeArrayDeviceView hits,
               const uint2 seed_range, const ParamsPOD params, const bool fw, const bool rc)
{ map_exact_t( read_batch, fmi, rfmi, hits, seed_range, params, fw, rc ); }
void map_approx(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi, SeedHitDequeArrayDeviceView hits,
                const uint2 seed_range, const ParamsPOD params, const bool fw, const bool rc)
{ map_approx_t( read_batch, fmi, rfmi, hits, seed_range, params, fw, rc ); }
void map_whole_read(const ReadsDef::type& read_batch, const FMIndexDef::type fmi, const FMIndexDef::type rfmi,
                    const nvbio::cuda::PingPongQueuesView<uint32> queues, uint8* reseed, SeedHitDequeArrayDeviceView hits,
                    const ParamsPOD params, const bool fw, const bool rc)
{ map_whole_read_t( read_batch, fmi, rfmi, queues, reseed, hits, params, fw, rc ); }
// gather_ranges (mapping.cu:36-81): out_ranges[t] = size of the t-th seed-hit range, reads in order, hits in deque order
inline __global__ void b200_gather_ranges_kernel(const uint32 count, const uint32 n_reads, const SeedHitDequeArrayDeviceView hits,
                                                 const uint32* hit_counts_scan, uint64* out_ranges)
{
    const uint32 t = threadIdx.x + blockDim.x * blockIdx.x;
    if (t >= count) return;
    uint32 lo = 0u, hi = n_reads;                                   // first read whose inclusive hit-count scan exceeds t
    while (lo < hi) { const uint32 mid = (lo + hi) >> 1; if (hit_counts_scan[mid] <= t) lo = mid + 1u; else hi = mid; }
    const uint32 first = lo ? hit_counts_scan[lo - 1u] : 0u;
    const uint2 range = hits.get_data( lo )[ t - first ].get_range();
    out_ranges[t] = range.y - range.x;
}
void gather_ranges(const uint32 count, const uint32 n_reads, const SeedHitDequeArrayDeviceView hits, const uint32* hit_counts_scan, uint64* out_ranges)
{
    if (count) b200_gather_ranges_kernel<<< (count + 127u) / 128u, 128u >>>( count, n_reads, hits, hit_counts_scan, out_ranges );
}
#endif // NVBIO_B200_DEFINE_NVBOWTIE_MAPPING

} // namespace cuda
} // namespace bowtie2
} // namespace nvbio
