// nvbio_b200/shim/batched_alignment.h -- nvbio::aln::BatchedBandedAlignmentScore / BatchedAlignmentScore for Gotoh aligners,
// forwarding enact() to the nvbio_b200 DP kernels (nvb_banded_gotoh_score / nvb_gotoh_score).
//
// What is replaced (reference tree):
//   BatchedBandedAlignmentScore<BAND_LEN,stream,DeviceThreadBlockScheduler<BD,MB>>::enact    nvbio/alignment/batched_banded_inl.h:135-162
//   BatchedBandedAlignmentScore<BAND_LEN,stream,DeviceStagedThreadScheduler>::enact          nvbio/alignment/batched_banded_inl.h:170-241
//   BatchedAlignmentScore<stream,DeviceThreadBlockScheduler<BD,MB>>::enact                   nvbio/alignment/batched_inl.h:329-440
//   and through them aln::batch_banded_alignment_score<BAND_LEN>() / aln::batch_alignment_score()   (batched_inl.h:984-1101)
// for every stream that is *bound*: b200::stream_binding<stream_type> tells the shim where the stream's packed strings
// live.  priv::AlignmentStream (the stream the convenience functions build, batched_inl.h:863-982) is bound here for
// every packed string-set type of views.h; a user stream is bound with a few lines (see tests/shim/shim_harness.cu).
//
// How a bound stream is run -- the stream concept (batched.h:239-309) stays in charge of everything but the DP:
//   1. b200::layout_kernel   calls stream.init_context(i) and reads the offset / length of pattern i and text i;
//   2. the C ABI call        scores all alignments (DPX s16x2 kernels; int32 kernels for what they do not admit);
//   3. b200::output_kernel   calls stream.init_context(i) again, feeds (score, sink) to the context's own sink with
//                            sink.report() and hands the context to stream.output(i) -- so BestSink<int16> scores,
//                            nvBowtie-style clamps or any other output rule of the stream are honoured unchanged.
// Anything that is not bound, is not a Gotoh aligner over SimpleGotohScheme, or does not keep a BestSink falls through
// to the reference's own kernel, at compile time.
#pragma once

#include <nvbio_b200/shim/views.h>
#include <nvbio/alignment/alignment.h>
#include <nvbio/alignment/batched.h>
#include <limits>

namespace nvbio {
namespace aln {
namespace b200 {

using nvbio::b200::check;
using nvbio::b200::stats;
using nvbio::b200::scratch;
using nvbio::b200::SCRATCH_LAYOUT; using nvbio::b200::SCRATCH_SCORE; using nvbio::b200::SCRATCH_SINK; using nvbio::b200::SCRATCH_TEMP;
using nvbio::b200::SCRATCH_PATTERNS; using nvbio::b200::SCRATCH_QUALS;

// ------------------------------------------------------------------------------------------------------
// customisation point: where do the strings of a stream live?
//   static const bool bound;
//   typedef ... pattern_string / text_string (packed strings, see views.h packed_string<>)
//   static const uint32* pattern_words(const stream&), text_words(const stream&)        (host)
//   static pattern_string pattern(const stream&, i, const context_type*), text(...)     (device)
// ------------------------------------------------------------------------------------------------------
template <typename stream_type> struct stream_binding { static const bool bound = false; };

/// defaults a binding inherits: the length bounds come from the stream itself (a binding may hide them, e.g. for a stream whose
/// own accessors do not compile: nvBowtie's BestScoreStream::max_pattern_length() calls a reads.max_read_len() that does not exist)
template <typename stream_type>
struct binding_defaults
{
    static uint32 max_pattern_length(const stream_type& s) { return s.max_pattern_length(); }
    static uint32 max_text_length   (const stream_type& s) { return s.max_text_length(); }
};

template <typename aligner_type, typename pattern_set, typename text_set, typename sink_iterator>
struct stream_binding< priv::AlignmentStream<aligner_type,pattern_set,trivial_quality_string_set,text_set,sink_iterator> > :
    public binding_defaults< priv::AlignmentStream<aligner_type,pattern_set,trivial_quality_string_set,text_set,sink_iterator> >
{
    typedef priv::AlignmentStream<aligner_type,pattern_set,trivial_quality_string_set,text_set,sink_iterator> stream_type;
    typedef typename stream_type::context_type      context_type;
    typedef typename pattern_set::string_type       pattern_string;
    typedef typename text_set::string_type          text_string;

    static const bool bound = nvbio::b200::packed_string_set<pattern_set>::supported &&
                              nvbio::b200::packed_string_set<text_set>::supported;

    static const uint32* pattern_words(const stream_type& s) { return nvbio::b200::packed_string_set<pattern_set>::words( s.m_patterns ); }
    static const uint32* text_words   (const stream_type& s) { return nvbio::b200::packed_string_set<text_set>::words( s.m_texts ); }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static pattern_string pattern(const stream_type& s, const uint32 i, const context_type*) { return s.m_patterns[i]; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE static text_string    text   (const stream_type& s, const uint32 i, const context_type*) { return s.m_texts[i]; }
};

// ------------------------------------------------------------------------------------------------------
// which aligners / sinks the DP kernels implement
// ------------------------------------------------------------------------------------------------------
template <typename aligner_type> struct gotoh_scheme_of { static const bool supported = false; };
template <AlignmentType TYPE_T, typename algorithm_tag>
struct gotoh_scheme_of< GotohAligner<TYPE_T,SimpleGotohScheme,algorithm_tag> >
{
    static const bool supported = true;
    static const int  TYPE      = int(TYPE_T);           // GLOBAL 0, LOCAL 1, SEMI_GLOBAL 2 == NVB_GLOBAL / NVB_LOCAL / NVB_SEMI_GLOBAL
    static nvb_gotoh_scheme get(const GotohAligner<TYPE_T,SimpleGotohScheme,algorithm_tag>& a)
    {
        nvb_gotoh_scheme s;
        s.match = a.scheme.m_match;               s.mismatch = a.scheme.m_mismatch;
        s.pattern_gap_open = a.scheme.m_gap_open; s.pattern_gap_ext = a.scheme.m_gap_ext;
        s.text_gap_open    = a.scheme.m_gap_open; s.text_gap_ext    = a.scheme.m_gap_ext;
        s.d_qual_table = NULL; s.qual_table_min = 0; s.qual_table_max = 0;
        return s;
    }
};
template <typename sink_type> struct is_best_sink                        { static const bool value = false; };
template <typename T>         struct is_best_sink< BestSink<T> >         { static const bool value = std::is_integral<T>::value; };

template <typename stream_type>
struct is_accelerated
{
    typedef typename stream_type::aligner_type  aligner_type;
    typedef typename stream_type::context_type  context_type;
    typedef typename std::decay< decltype( std::declval<context_type&>().sink ) >::type sink_type;
    static const bool value = stream_binding<stream_type>::bound &&
                              gotoh_scheme_of<aligner_type>::supported &&
                              is_best_sink<sink_type>::value;
};
/// Bounds of the DP values a batch can produce, from its scheme and the stream's length bounds: no H exceeds `hi` (a match, or the
/// best quality-table score, on every row), and no H, E or F of a real path falls below `lo` (the worst single cost on each of the at most
/// max_pattern_length + max_text_length steps, opening included).  `match` is the scheme's match(0), the reference's give-up rate.
struct score_range { int64 hi, lo, match; };

template <typename stream_type>
score_range score_range_of(const stream_type& stream)
{
    typedef typename stream_type::aligner_type aligner_type;
    const nvb_gotoh_scheme s = gotoh_scheme_of<aligner_type>::get( stream.aligner() );
    const int64 best  = nvbio::max( nvbio::max( int64( s.match ), int64( 0 ) ), int64( s.d_qual_table ? s.qual_table_max : 0 ) );
    const int64 worst = nvbio::min( nvbio::min( nvbio::min( int64( s.mismatch ), int64( 0 ) ), int64( s.d_qual_table ? s.qual_table_min : 0 ) ),
                                    nvbio::min( nvbio::min( int64( s.pattern_gap_open ), int64( s.pattern_gap_ext ) ),
                                                nvbio::min( int64( s.text_gap_open ), int64( s.text_gap_ext ) ) ) );
    const int64 max_p = stream_binding<stream_type>::max_pattern_length( stream ), max_t = stream_binding<stream_type>::max_text_length( stream );
    score_range r; r.hi = best * max_p; r.lo = 2 * worst * (max_p + max_t); r.match = s.match;
    return r;
}

/// A sink narrower than int32 (BestSink<int16>): the reference computes int32 cell scores and reports them through the sink's own
/// type -- LOCAL every cell, SEMI_GLOBAL every cell of the last row, GLOBAL one cell -- keeping the best of the NARROWED values, while
/// the engine reports the int32 best once.  The two agree when every score the alignment type can report fits the sink's type
/// (GLOBAL always: one report either way; LOCAL reports no negative score); a batch whose bounds allow more runs the reference's kernel.
template <typename stream_type>
struct sink_fits
{
    typedef typename stream_type::aligner_type  aligner_type;
    typedef typename stream_type::context_type  context_type;
    typedef typename std::decay< decltype( std::declval<context_type&>().sink.score ) >::type score_type;

    static bool check(const stream_type& stream)
    {
        if (sizeof(score_type) >= sizeof(int32) || gotoh_scheme_of<aligner_type>::TYPE == int(GLOBAL)) return true;
        const score_range r = score_range_of( stream );
        const int64 lo = gotoh_scheme_of<aligner_type>::TYPE == int(LOCAL) ? 0 : r.lo;
        return r.hi <= int64( std::numeric_limits<score_type>::max() ) && lo >= int64( std::numeric_limits<score_type>::min() );
    }
};

/// flag[0] |= 1 if some alignment's context.min_score could make the reference's staged unit give up on it: after a window that ends
/// before the pattern does, it stops when the band's best H < min_score + remaining rows x match (gotoh_banded_inl.h:622-633).  The
/// band's best H is at least `lo`, so an alignment with min_score + pattern_length x match <= lo is never given up on.
template <typename stream_type>
__global__ void give_up_kernel(const stream_type stream, const int64 lo, const int64 match, uint32* flag)
{
    typedef typename stream_type::context_type context_type;
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= stream.size()) return;
    context_type context;
    if (stream.init_context( i, &context ) &&
        int64( context.min_score ) + int64( stream.pattern_length( i, &context ) ) * match > lo)
        atomicOr( flag, 1u );
}

/// DeviceStagedThreadScheduler: the reference scores 32-row windows (batched_stream.h:128,161-176) and carries the band between them in
/// short2 checkpoints (utils.h:52, gotoh_banded_inl.h:177-184), which wrap any H or F outside the int16 range, and it gives up on an
/// alignment whose min_score is out of reach.  The engine's single pass equals those passes when neither can happen: every H, E and F
/// of a real path within [SHRT_MIN + 32, 32767], and no min_score in reach of a give-up.  Anything else runs the reference's kernel.
template <typename stream_type>
struct staged_fits
{
    static bool check(const stream_type& stream)
    {
        const score_range r = score_range_of( stream );
        if (r.hi > 32767 || r.lo < int64( std::numeric_limits<int16>::min() ) + 32) return false;
        const uint32 n = stream.size();
        if (n == 0u) return true;
        uint32* d_flag = (uint32*)scratch( SCRATCH_SCORE, sizeof(uint32) );
        uint32  h_flag = 0u;
        check_cuda( cudaMemset( d_flag, 0, sizeof(uint32) ), "cudaMemset" );
        give_up_kernel<<<(n + 127u) / 128u,128>>>( stream, r.lo, r.match, d_flag );
        check_cuda( cudaMemcpy( &h_flag, d_flag, sizeof(uint32), cudaMemcpyDeviceToHost ), "cudaMemcpy" );
        return h_flag == 0u;
    }
private:
    static void check_cuda(const cudaError_t e, const char* what) { if (e != cudaSuccess) nvbio::b200::check( NVB_E_INVALID, what ); }
};
template <typename stream_type, typename scheduler_type>
struct scheduler_fits { static bool check(const stream_type&) { return true; } };
template <typename stream_type>
struct scheduler_fits<stream_type, DeviceStagedThreadScheduler> { static bool check(const stream_type& s) { return staged_fits<stream_type>::check( s ); } };

template <uint32 BAND_LEN> struct is_band_supported
{
    static const bool value = (BAND_LEN == 3u || BAND_LEN == 5u || BAND_LEN == 7u || BAND_LEN == 15u || BAND_LEN == 31u || BAND_LEN == 63u);
};

// ------------------------------------------------------------------------------------------------------
// step 1 and step 3
// ------------------------------------------------------------------------------------------------------
template <typename stream_type>
__global__ void layout_kernel(const stream_type stream, uint32* p_off, uint32* p_len, uint32* t_off, uint32* t_len)
{
    typedef stream_binding<stream_type>             binding;
    typedef typename stream_type::context_type      context_type;
    typedef typename binding::pattern_string        pattern_string;
    typedef typename binding::text_string           text_string;
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= stream.size()) return;
    context_type context;
    uint32 po = 0u, pl = 0u, to = 0u, tl = 0u;
    if (stream.init_context( i, &context ))
    {
        const pattern_string p = binding::pattern( stream, i, &context );
        const text_string    t = binding::text( stream, i, &context );
        po = nvbio::b200::packed_string<pattern_string>::offset( p ); pl = nvbio::b200::packed_string<pattern_string>::length( p );
        to = nvbio::b200::packed_string<text_string>::offset( t );    tl = nvbio::b200::packed_string<text_string>::length( t );
    }
    p_off[i] = po; p_len[i] = pl; t_off[i] = to; t_len[i] = tl;
}

template <typename stream_type>
__global__ void output_kernel(const stream_type stream, const int32* score, const uint2* sink)
{
    typedef typename stream_type::context_type      context_type;
    typedef typename std::decay< decltype( std::declval<context_type&>().sink.score ) >::type score_type;
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= stream.size()) return;
    context_type context;
    if (stream.init_context( i, &context ))
    {
        const uint2 k = sink[i];
        if (k.x != 0xFFFFFFFFu)                             // (-1,-1): the DP did not run (text shorter than pattern), sink left at its defaults
            context.sink.report( score_type( score[i] ), k );
    }
    stream.output( i, &context );
}

// a binding may declare `static const bool materialise_patterns = true`: its patterns are not plain substrings of a packed stream
// (e.g. nvBowtie reads them reversed and / or complemented through a ReadLoader) -- then the engine calls the stream's OWN
// load_strings() once per alignment and writes pattern symbols and base qualities to byte buffers the DP kernels read
template <typename binding, typename = void> struct materialises_patterns { static const bool value = false; };
template <typename binding> struct materialises_patterns<binding, typename std::enable_if<binding::materialise_patterns>::type> { static const bool value = true; };

template <typename stream_type>
__global__ void materialise_kernel(const stream_type stream, const uint32 p_stride, uint8* pat, uint8* qual,
                                   uint32* p_off, uint32* p_len, uint32* t_off, uint32* t_len)
{
    typedef stream_binding<stream_type>             binding;
    typedef typename stream_type::context_type      context_type;
    typedef typename stream_type::strings_type      strings_type;
    typedef typename binding::text_string           text_string;
    const uint32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= stream.size()) return;
    context_type context;
    uint32 pl = 0u, to = 0u, tl = 0u;
    if (stream.init_context( i, &context ))
    {
        pl = stream.pattern_length( i, &context );
        strings_type strings;
        stream.load_strings( i, 0u, pl, &context, &strings );
        // four symbols per store (p_stride is a multiple of 4 and the buffers are word aligned)
        uint32* p = reinterpret_cast<uint32*>( pat  + size_t(i) * p_stride );
        uint32* q = reinterpret_cast<uint32*>( qual + size_t(i) * p_stride );
        for (uint32 j = 0; j < pl; j += 4u)
        {
            uint32 pw = 0u, qw = 0u;
            for (uint32 k = 0; k < 4u; ++k)
                if (j + k < pl) { pw |= uint32( uint8( strings.pattern[j + k] ) ) << (8u * k); qw |= uint32( uint8( strings.quals[j + k] ) ) << (8u * k); }
            p[j >> 2] = pw; q[j >> 2] = qw;
        }
        const text_string t = binding::text( stream, i, &context );
        to = nvbio::b200::packed_string<text_string>::offset( t ); tl = nvbio::b200::packed_string<text_string>::length( t );
    }
    p_off[i] = i * p_stride; p_len[i] = pl; t_off[i] = to; t_len[i] = tl;
}

/// the common body of the accelerated enact() functions
template <typename stream_type>
struct engine
{
    typedef stream_binding<stream_type>                     binding;
    typedef typename stream_type::aligner_type              aligner_type;
    typedef gotoh_scheme_of<aligner_type>                   scheme_of;
    typedef typename binding::text_string                   text_string;
    static const bool MATERIALISE = materialises_patterns<binding>::value;

    /// band_len == 0: full matrix
    void enact(const stream_type& stream, const uint32 band_len)
    {
        const uint32 n = stream.size();
        if (n == 0u) return;
        uint32* p_off = (uint32*)scratch( SCRATCH_LAYOUT, 4u * size_t(n) * sizeof(uint32) );
        uint32* p_len = p_off + n; uint32* t_off = p_len + n; uint32* t_len = t_off + n;
        const uint32 grid = (n + 127u) / 128u;

        nvb_string_set P, T;
        const uint8_t* d_quals = NULL;
        stage( stream, grid, p_off, p_len, t_off, t_len, P, d_quals, std::integral_constant<bool,MATERIALISE>() );
        P.d_offsets = p_off; P.d_lengths = p_len; P.stride = 0u; P.length = binding::max_pattern_length( stream );
        T.d_words = (const uint32_t*)binding::text_words( stream );
        T.bits = nvbio::b200::packed_string<text_string>::BITS;    T.big_endian = nvbio::b200::packed_string<text_string>::BE;
        T.d_offsets = t_off; T.d_lengths = t_len; T.stride = 0u; T.length = binding::max_text_length( stream );

        const nvb_gotoh_scheme scheme = scheme_of::get( stream.aligner() );
        int32_t*   d_score = (int32_t*)scratch( SCRATCH_SCORE, size_t(n) * sizeof(int32_t) );
        nvb_uint2* d_sink  = (nvb_uint2*)scratch( SCRATCH_SINK, size_t(n) * sizeof(nvb_uint2) );
        size_t bytes = 0u;
        int r = band_len ? nvb_banded_gotoh_score( int(band_len), scheme_of::TYPE, &scheme, &P, d_quals, &T, n, d_score, d_sink, NULL, &bytes, NULL )
                         : nvb_gotoh_score( scheme_of::TYPE, &scheme, &P, d_quals, &T, n, d_score, d_sink, NULL, &bytes, NULL );
        if (r != NVB_E_TEMP_SIZE) check( r, "DP temp size query" );
        void* d_temp = scratch( SCRATCH_TEMP, bytes + 256u );
        bytes += 256u;
        r = band_len ? nvb_banded_gotoh_score( int(band_len), scheme_of::TYPE, &scheme, &P, d_quals, &T, n, d_score, d_sink, d_temp, &bytes, NULL )
                     : nvb_gotoh_score( scheme_of::TYPE, &scheme, &P, d_quals, &T, n, d_score, d_sink, d_temp, &bytes, NULL );
        check( r, band_len ? "nvb_banded_gotoh_score" : "nvb_gotoh_score" );

        output_kernel<<<grid,128>>>( stream, (const int32*)d_score, (const uint2*)d_sink );
        if (band_len) stats().banded_score++; else stats().full_score++;
    }

private:
    // patterns readable in place
    void stage(const stream_type& stream, const uint32 grid, uint32* p_off, uint32* p_len, uint32* t_off, uint32* t_len,
               nvb_string_set& P, const uint8_t*& d_quals, std::false_type)
    {
        typedef typename binding::pattern_string pattern_string;
        layout_kernel<<<grid,128>>>( stream, p_off, p_len, t_off, t_len );
        P.d_words = (const uint32_t*)binding::pattern_words( stream );
        P.bits = nvbio::b200::packed_string<pattern_string>::BITS; P.big_endian = nvbio::b200::packed_string<pattern_string>::BE;
        d_quals = NULL;
    }
    // patterns (and qualities) copied out through the stream's own loaders
    void stage(const stream_type& stream, const uint32 grid, uint32* p_off, uint32* p_len, uint32* t_off, uint32* t_len,
               nvb_string_set& P, const uint8_t*& d_quals, std::true_type)
    {
        const uint32 p_stride = (binding::max_pattern_length( stream ) + 3u) & ~3u;
        uint8* d_pat  = (uint8*)scratch( SCRATCH_PATTERNS, size_t(stream.size()) * p_stride + 16u );
        uint8* d_qual = (uint8*)scratch( SCRATCH_QUALS,    size_t(stream.size()) * p_stride + 16u );
        materialise_kernel<<<grid,128>>>( stream, p_stride, d_pat, d_qual, p_off, p_len, t_off, t_len );
        P.d_words = (const uint32_t*)d_pat;
        P.bits = 8u; P.big_endian = 0u;
        d_quals = d_qual;
    }
};

struct no_engine {};

/// A stream that behaves exactly like `stream_type` but is a different type: instantiating the reference's batch classes
/// on it reaches the reference's own (generic) partial specialisations instead of the ones below -- the compile-time
/// fall-back for everything the nvbio_b200 kernels do not cover.
template <typename stream_type>
struct unbound_stream : public stream_type
{
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE unbound_stream(const stream_type& s) : stream_type( s ) {}
};

/// Base class for the partial specialisations below and for a user-written one that binds a stream TEMPLATE of their own:
///   template <uint32 BD, uint32 MB, uint32 BAND_LEN, ...>
///   struct BatchedBandedAlignmentScore<BAND_LEN, MyStream<...>, DeviceThreadBlockScheduler<BD,MB> > :
///       public b200::BandedScoreBatch<BAND_LEN, MyStream<...>, DeviceThreadBlockScheduler<BD,MB> > {};
/// (plus a stream_binding<MyStream<...>> specialisation).  An instantiation the kernels do not cover runs the reference's.
template <uint32 BAND_LEN, typename stream_type, typename scheduler_type>
struct BandedScoreBatch
{
    typedef BatchedBandedAlignmentScore<BAND_LEN, unbound_stream<stream_type>, scheduler_type>   reference_batch;
    typedef typename stream_type::aligner_type                                                  aligner_type;
    typedef typename reference_batch::cell_type                                                 cell_type;
    static const bool accelerated = is_accelerated<stream_type>::value && is_band_supported<BAND_LEN>::value;

    // the reference's temp-storage contract (batched_banded_inl.h:141-147, 180-199), so that callers sizing buffers see the same numbers
    static uint64 min_temp_storage(const uint32 mp, const uint32 mt, const uint32 n) { return reference_batch::min_temp_storage( mp, mt, n ); }
    static uint64 max_temp_storage(const uint32 mp, const uint32 mt, const uint32 n) { return reference_batch::max_temp_storage( mp, mt, n ); }

    /// enact the batch execution (the DPX kernels manage their own scratch; `temp` is only used by the fall-back)
    void enact(stream_type stream, uint64 temp_size = 0u, uint8* temp = NULL)
    {
        run( stream, temp_size, temp, std::integral_constant<bool,accelerated>() );
    }
private:
    void run(const stream_type& stream, uint64 temp_size, uint8* temp, std::true_type)
    {
        if (sink_fits<stream_type>::check( stream ) && scheduler_fits<stream_type,scheduler_type>::check( stream )) m_engine.enact( stream, BAND_LEN );
        else                                         run( stream, temp_size, temp, std::false_type() );
    }
    void run(const stream_type& stream, uint64 temp_size, uint8* temp, std::false_type)
    {
        m_reference.enact( unbound_stream<stream_type>( stream ), temp_size, temp );
        stats().fallbacks++;
    }
    typename std::conditional<accelerated, engine<stream_type>, no_engine>::type m_engine;
    reference_batch     m_reference;
};

/// the same for the full-matrix batch class
template <typename stream_type, typename scheduler_type>
struct ScoreBatch
{
    typedef BatchedAlignmentScore<unbound_stream<stream_type>, scheduler_type>  reference_batch;
    typedef typename stream_type::aligner_type                                  aligner_type;
    typedef typename reference_batch::cell_type                                 cell_type;
    static const bool accelerated = is_accelerated<stream_type>::value;

    static uint64 min_temp_storage(const uint32 mp, const uint32 mt, const uint32 n) { return reference_batch::min_temp_storage( mp, mt, n ); }
    static uint64 max_temp_storage(const uint32 mp, const uint32 mt, const uint32 n) { return reference_batch::max_temp_storage( mp, mt, n ); }

    void enact(stream_type stream, uint64 temp_size = 0u, uint8* temp = NULL)
    {
        run( stream, temp_size, temp, std::integral_constant<bool,accelerated>() );
    }
private:
    void run(const stream_type& stream, uint64 temp_size, uint8* temp, std::true_type)
    {
        if (sink_fits<stream_type>::check( stream )) m_engine.enact( stream, 0u );
        else                                         run( stream, temp_size, temp, std::false_type() );
    }
    void run(const stream_type& stream, uint64 temp_size, uint8* temp, std::false_type)
    {
        m_reference.enact( unbound_stream<stream_type>( stream ), temp_size, temp );
        stats().fallbacks++;
    }
    typename std::conditional<accelerated, engine<stream_type>, no_engine>::type m_engine;
    reference_batch     m_reference;
};

} // namespace b200

// ------------------------------------------------------------------------------------------------------
// the partial specialisations proper: the streams the convenience functions build over string sets
// (aln::batch_banded_alignment_score<BAND_LEN>(), aln::batch_alignment_score(); batched_inl.h:984-1101)
// ------------------------------------------------------------------------------------------------------

/// banded, thread scheduler (batched_banded_inl.h:135-162)
template <uint32 BLOCKDIM, uint32 MINBLOCKS, uint32 BAND_LEN,
          AlignmentType TYPE, typename algorithm_tag, typename pattern_set, typename text_set, typename sink_iterator>
struct BatchedBandedAlignmentScore<
    BAND_LEN,
    priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,algorithm_tag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
    DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > :
    public b200::BandedScoreBatch<
        BAND_LEN,
        priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,algorithm_tag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
        DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > {};

/// banded, staged scheduler (batched_banded_inl.h:170-241): the DPX kernels need no staging, every alignment is scored in one pass,
/// which equals the reference's windowed passes where staged_fits holds (no int16 wrap in its checkpoints, no give-up on min_score);
/// other batches run the reference's staged kernel
template <uint32 BAND_LEN,
          AlignmentType TYPE, typename algorithm_tag, typename pattern_set, typename text_set, typename sink_iterator>
struct BatchedBandedAlignmentScore<
    BAND_LEN,
    priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,algorithm_tag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
    DeviceStagedThreadScheduler > :
    public b200::BandedScoreBatch<
        BAND_LEN,
        priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,algorithm_tag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
        DeviceStagedThreadScheduler > {};

/// full matrix, thread scheduler (batched_inl.h:329-440)
template <uint32 BLOCKDIM, uint32 MINBLOCKS,
          AlignmentType TYPE, typename pattern_set, typename text_set, typename sink_iterator>
struct BatchedAlignmentScore<
    priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,PatternBlockingTag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
    DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > :
    public b200::ScoreBatch<
        priv::AlignmentStream< GotohAligner<TYPE,SimpleGotohScheme,PatternBlockingTag>, pattern_set, trivial_quality_string_set, text_set, sink_iterator >,
        DeviceThreadBlockScheduler<BLOCKDIM,MINBLOCKS> > {};

} // namespace aln
} // namespace nvbio
