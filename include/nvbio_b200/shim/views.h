// nvbio_b200/shim/views.h -- compile-time extraction of raw device views from nvbio's own iterator / string-set /
// FM-index types, so that the reference's templates can forward to the C ABI of include/nvbio_b200.h.
//
// Everything here is a trait: a type the shim does not recognise has `supported == false` and the caller keeps the
// reference template's own code path (decided at compile time; there is no run-time CPU fallback).
// Types follow the reference tree:
//   cuda::ldg_pointer<T>                        nvbio/basic/cuda/ldg.h:44-360          (m_base)
//   PackedStream<It,Sym,BITS,BE,Index>          nvbio/basic/packedstream.h:190-328     (stream(), index())
//   deinterleaved_iterator<STRIDE,WHICH,It>     nvbio/basic/deinterleaved_iterator.h:39-184 (m_it)
//   ConcatenatedStringSet / SparseStringSet     nvbio/strings/string_set.h:480-553, 613-686
//   InfixSet                                    nvbio/strings/infix.h:320-422, 541-590
//   fm_index / rank_dictionary / SSA context    nvbio/fmindex/fmindex.h:341-387, rank_dictionary.h:82-134, ssa.h:220-247
#pragma once

#include <nvbio_b200.h>
#include <nvbio/basic/types.h>
#include <nvbio/basic/packedstream.h>
#include <nvbio/basic/deinterleaved_iterator.h>
#include <nvbio/basic/cuda/ldg.h>
#include <nvbio/basic/vector_view.h>
#include <nvbio/strings/string_set.h>
#include <nvbio/strings/infix.h>
#include <nvbio/fmindex/fmindex.h>
#include <nvbio/fmindex/ssa.h>
#include <thrust/device_vector.h>
#include <cuda_runtime.h>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>

namespace nvbio {
namespace b200 {

/// the analogue of the reference's cuda::check_error exceptions for the C ABI's return codes
inline void check(const int err, const char* what)
{
    if (err != NVB_OK)
        throw std::runtime_error( std::string("nvbio_b200: ") + what + ": " + nvb_error_string( err ) );
}

/// counters of the calls that went through the nvbio_b200 kernels (so that a harness can prove which path ran)
struct shim_stats
{
    uint64 fm_rank, fm_locate, banded_score, full_score, fallbacks;
};
inline shim_stats& stats() { static shim_stats s = { 0u, 0u, 0u, 0u, 0u }; return s; }

// ------------------------------------------------------------------------------------------------------
// grow-only device scratch, one arena per (host thread, slot).  The reference's convenience functions construct a batch object per
// call (batched_inl.h:984-1101) and thrust::device_vector members would cost a cudaMalloc + cudaFree each, which is more than
// the DP of a small batch takes.  Every shim launch goes to the legacy default stream, so consecutive calls that reuse an arena are
// ordered; growing an arena goes through cudaFree, which synchronises.  The arenas are released at process exit by the driver.
// ------------------------------------------------------------------------------------------------------
enum scratch_slot { SCRATCH_LAYOUT = 0, SCRATCH_SCORE, SCRATCH_SINK, SCRATCH_TEMP, SCRATCH_PATTERNS, SCRATCH_QUALS, SCRATCH_TABLE, SCRATCH_SLOTS };

inline void* scratch(const scratch_slot slot, const size_t bytes)
{
    struct arena { void* ptr; size_t bytes; int device; };
    static thread_local arena arenas[SCRATCH_SLOTS] = {};
    int device = 0;
    if (cudaGetDevice( &device ) != cudaSuccess) check( NVB_E_INVALID, "cudaGetDevice" );
    arena& a = arenas[slot];
    if (a.ptr == NULL || a.device != device || a.bytes < bytes)
    {
        if (a.ptr)
        {
            if (a.device != device) { cudaSetDevice( a.device ); cudaFree( a.ptr ); cudaSetDevice( device ); }
            else                      cudaFree( a.ptr );
            a.ptr = NULL; a.bytes = 0u;
        }
        size_t cap = bytes + bytes / 2u;
        if (cap < (size_t(1u) << 16)) cap = size_t(1u) << 16;
        cap = (cap + 255u) & ~size_t(255u);
        if (cudaMalloc( &a.ptr, cap ) != cudaSuccess)
        {
            cudaGetLastError();
            cap = (bytes + 255u) & ~size_t(255u);
            if (cudaMalloc( &a.ptr, cap ) != cudaSuccess) { a.ptr = NULL; check( NVB_E_INVALID, "device scratch allocation" ); }
        }
        a.bytes = cap; a.device = device;
    }
    return a.ptr;
}
template <typename T> inline T* scratch(const scratch_slot slot, const size_t count, const T*) { return (T*)scratch( slot, count * sizeof(T) ); }

// ------------------------------------------------------------------------------------------------------
// word iterators whose raw device pointer can be recovered
// ------------------------------------------------------------------------------------------------------
template <typename It> struct word_pointer { static const bool supported = false; typedef void value_type; };
template <typename T> struct word_pointer<const T*>
{
    static const bool supported = true; typedef T value_type;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const T* get(const T* p) { return p; }
};
template <typename T> struct word_pointer<T*>
{
    static const bool supported = true; typedef T value_type;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const T* get(const T* p) { return p; }
};
template <typename T> struct word_pointer< cuda::ldg_pointer<T> >
{
    static const bool supported = true; typedef T value_type;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const T* get(const cuda::ldg_pointer<T>& p) { return p.m_base; }
};

// ------------------------------------------------------------------------------------------------------
// packed symbol iterators: PackedStream over 32-bit words, 2 or 4 bits per symbol
// ------------------------------------------------------------------------------------------------------
template <typename T> struct packed_iterator
{
    static const bool   supported = false;
    static const uint32 BITS = 0u;
    static const uint32 BE   = 0u;
};
template <typename It, typename Sym, uint32 BITS_T, bool BE_T>
struct packed_iterator< PackedStream<It,Sym,BITS_T,BE_T,uint32> >
{
    typedef PackedStream<It,Sym,BITS_T,BE_T,uint32> type;
    static const bool   supported = word_pointer<It>::supported &&
                                    std::is_same<typename std::remove_cv<typename word_pointer<It>::value_type>::type,uint32>::value &&
                                    (BITS_T == 2u || BITS_T == 4u);
    static const uint32 BITS = BITS_T;
    static const uint32 BE   = BE_T ? 1u : 0u;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const uint32* words(const type& s) { return (const uint32*)word_pointer<It>::get( s.stream() ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static uint32        offset(const type& s) { return s.index(); }
};

// ------------------------------------------------------------------------------------------------------
// strings over a supported packed iterator: vector_view<PackedStream> and Infix<string, coords>
// (only __host__ __device__ members of the reference types are used: Infix::begin() is host-only, infix.h:229-245)
// ------------------------------------------------------------------------------------------------------
template <typename S> struct packed_string
{
    static const bool   supported = false;
    static const uint32 BITS = 0u;
    static const uint32 BE   = 0u;
};
template <typename It, typename Index>
struct packed_string< vector_view<It,Index> >
{
    typedef vector_view<It,Index>   type;
    typedef packed_iterator<It>     traits;
    static const bool   supported = traits::supported;
    static const uint32 BITS = traits::BITS;
    static const uint32 BE   = traits::BE;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const uint32* words(const type& s)  { return traits::words( s.begin() ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static uint32        offset(const type& s) { return traits::offset( s.begin() ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static uint32        length(const type& s) { return uint32( s.size() ); }
};
template <typename StringType, typename CoordType>
struct packed_string< Infix<StringType,CoordType> >
{
    typedef Infix<StringType,CoordType> type;
    typedef packed_string<StringType>   base;
    static const bool   supported = base::supported;
    static const uint32 BITS = base::BITS;
    static const uint32 BE   = base::BE;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static const uint32* words(const type& s)  { return base::words( s.m_string ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static uint32        offset(const type& s) { return base::offset( s.m_string ) + uint32( s.range().x ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static uint32        length(const type& s) { return uint32( s.size() ); }
};

// ------------------------------------------------------------------------------------------------------
// string sets: the word pointer all their strings share, recovered on the HOST from the set object
// (the per-string offsets and lengths are read on the device by a small kernel through set[i])
// ------------------------------------------------------------------------------------------------------
template <typename Set> struct packed_string_set { static const bool supported = false; static const uint32 BITS = 0u; static const uint32 BE = 0u; };

template <typename SI, typename OI>
struct packed_string_set< ConcatenatedStringSet<SI,OI> >
{
    typedef ConcatenatedStringSet<SI,OI> type;
    static const bool   supported = packed_iterator<SI>::supported;
    static const uint32 BITS = packed_iterator<SI>::BITS;
    static const uint32 BE   = packed_iterator<SI>::BE;
    static const uint32* words(const type& set) { return packed_iterator<SI>::words( set.base_string() ); }
};
template <typename SI, typename RI>
struct packed_string_set< SparseStringSet<SI,RI> >
{
    typedef SparseStringSet<SI,RI> type;
    static const bool   supported = packed_iterator<SI>::supported;
    static const uint32 BITS = packed_iterator<SI>::BITS;
    static const uint32 BE   = packed_iterator<SI>::BE;
    static const uint32* words(const type& set) { return packed_iterator<SI>::words( set.base_string() ); }
};
// a single packed string used as the "sequence" of an InfixSet (infixes of one long string, e.g. a genome)
template <typename SI>
struct packed_string_set< vector_view<SI> >
{
    typedef vector_view<SI> type;
    static const bool   supported = packed_iterator<SI>::supported;
    static const uint32 BITS = packed_iterator<SI>::BITS;
    static const uint32 BE   = packed_iterator<SI>::BE;
    static const uint32* words(const type& s) { return packed_iterator<SI>::words( s.begin() ); }
};
// infixes of a string or of a string set (the seed sets built by extract_seeds-style code)
template <typename Seq, typename II>
struct packed_string_set< InfixSet<Seq,II> >
{
    typedef InfixSet<Seq,II> type;
    static const bool   supported = packed_string_set<Seq>::supported;
    static const uint32 BITS = packed_string_set<Seq>::BITS;
    static const uint32 BE   = packed_string_set<Seq>::BE;
    static const uint32* words(const type& set) { return packed_string_set<Seq>::words( set.m_sequence ); }
};

/// offsets[i], lengths[i] of every string of a set, read through the set's own operator[] on the device
template <typename Set>
__global__ void string_set_layout_kernel(const Set set, const uint32 n, uint32* offsets, uint32* lengths)
{
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typedef typename Set::string_type string_type;
    const string_type s = set[i];
    offsets[i] = packed_string<string_type>::offset( s );
    lengths[i] = packed_string<string_type>::length( s );
}

/// raw pointer of a thrust iterator / raw pointer naming device memory
template <typename It>
inline auto raw_device_pointer(It it) -> decltype( thrust::raw_pointer_cast( &*it ) ) { return thrust::raw_pointer_cast( &*it ); }

// ------------------------------------------------------------------------------------------------------
// FM-index: the production layout (interleaved {bwt,occ} uint4 pairs, SSA context) -> nvb_fm_index
// ------------------------------------------------------------------------------------------------------
template <typename FMI> struct fm_index_view { static const bool supported = false; };

template <typename BwtOccPtr, typename CountTable, uint32 SA_INT, typename SsaPtr>
struct fm_index_view<
    fm_index<
        rank_dictionary< 2u, 64u,
            PackedStream< deinterleaved_iterator<2,0,BwtOccPtr>, uint8, 2u, true, uint32 >,
            deinterleaved_iterator<2,1,BwtOccPtr>,
            CountTable >,
        SSA_index_multiple_context<SA_INT,SsaPtr>,
        null_type > >
{
    typedef fm_index<
        rank_dictionary< 2u, 64u,
            PackedStream< deinterleaved_iterator<2,0,BwtOccPtr>, uint8, 2u, true, uint32 >,
            deinterleaved_iterator<2,1,BwtOccPtr>,
            CountTable >,
        SSA_index_multiple_context<SA_INT,SsaPtr>,
        null_type >                                                     type;

    static const bool supported = word_pointer<BwtOccPtr>::supported && word_pointer<SsaPtr>::supported &&
                                  (SA_INT & (SA_INT - 1u)) == 0u;

    /// h_L2: the five words of the index's L2 table (device memory in the reference; the C ABI takes them by value)
    static nvb_fm_index get(const type& f)
    {
        nvb_fm_index v;
        v.d_bwt_occ   = (const void*)word_pointer<BwtOccPtr>::get( f.m_rank_dict.m_text.stream().m_it );
        v.d_ssa       = (const uint32_t*)word_pointer<SsaPtr>::get( f.m_sa.m_ssa );
        v.length      = f.m_length;
        v.primary     = f.m_primary;
        v.sa_interval = SA_INT;
        v.d_ktab      = NULL;
        v.ktab_k      = 0u;
        v.ktab_located = 0u;
        v.d_rows      = NULL;
        cudaPointerAttributes attr;
        const bool on_device = cudaPointerGetAttributes( &attr, f.m_L2 ) == cudaSuccess &&
                               (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
        if (on_device)
        {
            if (cudaMemcpy( v.L2, f.m_L2, 5u * sizeof(uint32), cudaMemcpyDeviceToHost ) != cudaSuccess)
                throw std::runtime_error( "nvbio_b200: cannot read the FM-index L2 table" );
        }
        else
        {
            (void)cudaGetLastError();
            for (uint32 i = 0; i < 5u; ++i) v.L2[i] = f.m_L2[i];
        }
        return v;
    }
};

} // namespace b200
} // namespace nvbio
