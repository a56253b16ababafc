// oracle/ref_shim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Thin extern "C" wrappers that instantiate the UNMODIFIED reference templates of
// NVlabs/nvbio (header-only, found under /root/reference at build time) on the host, so that
// tests and the CPU baseline can call the reference's own implementation of the two hot paths.
// Nothing from the reference is copied here: this file only *includes* the reference headers
// where they lie and calls their public entry points:
//
//   nvbio::gen_sa / gen_bwt_from_sa            nvbio/fmindex/bwt.h:38-63
//   nvbio::build_occurrence_table<2,64>        nvbio/fmindex/rank_dictionary_inl.h:42-77
//   nvbio::rank / match / locate               nvbio/fmindex/fmindex_inl.h:36-99, 280-341, 471-499
//   nvbio::SSA_index_multiple<16>              nvbio/fmindex/ssa_inl.h:262-277
//   nvbio::aln::banded_alignment_score<B>      nvbio/alignment/banded_inl.h:50-73
//                                              -> gotoh/gotoh_banded_inl.h:406-658
//
// Built by oracle/Makefile into oracle/_ref/libnvbio_ref.so (git-ignored build product).
// Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may load it.

#include <nvbio/basic/types.h>
#include <nvbio/basic/numbers.h>
#include <nvbio/basic/packedstream.h>
#include <nvbio/basic/deinterleaved_iterator.h>
#include <nvbio/basic/vector_view.h>
#include <nvbio/fmindex/bwt.h>
#include <nvbio/fmindex/ssa.h>
#include <nvbio/fmindex/fmindex.h>
#include <nvbio/alignment/alignment.h>
#include <nvbio/alignment/utils.h>
#include <vector>
#include <climits>
#include <cstring>
#include <omp.h>

using namespace nvbio;

namespace {

// production index layout (nvbio/io/fmindex/fmindex.h:302-319) with plain host pointers
typedef const uint4*                                               bwt_occ_ptr;
typedef deinterleaved_iterator<2,0,bwt_occ_ptr>                    bwt_iter;
typedef deinterleaved_iterator<2,1,bwt_occ_ptr>                    occ_iter;
typedef PackedStream<bwt_iter,uint8,2u,true>                       bwt_stream;
typedef rank_dictionary<2u,64u,bwt_stream,occ_iter,const uint32*>  rank_dict_t;
typedef SSA_index_multiple_context<16u,const uint32*>              ssa_ctx_t;
typedef fm_index<rank_dict_t,ssa_ctx_t>                            fm_index_t;

fm_index_t make_index(const uint32* bwt_occ, const uint32* ssa, const uint32* L2,
                      const uint32* count_table, uint32 n, uint32 primary)
{
    const bwt_occ_ptr p = (const uint4*)bwt_occ;
    return fm_index_t( n, primary, L2,
        rank_dict_t( bwt_stream( bwt_iter(p) ), occ_iter(p), count_table ),
        ssa_ctx_t( ssa ) );
}

typedef vector_view<const uint8*> str_view;

// a table-driven Gotoh scheme for the reference templates (a model of the GotohScoringScheme concept, nvbio/alignment/utils.h:
// 111-135): substitution scores by the pattern base's quality, table[2*q] on a match and table[2*q+1] on a mismatch -- the shape of
// nvBowtie's SmithWatermanScoringScheme<QualCost,...> (scoring.h:203-317) once its float expressions are evaluated on the host
struct TableGotohScheme
{
    const int32* tab; int32 pgo, pge, tgo, tge;
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 match(const uint8 q = 0)      const { return tab[2*q]; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 mismatch(const uint8 q = 0)   const { return tab[2*q+1]; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 mismatch(const uint8 a, const uint8 b, const uint8 q = 0) const { return tab[2*q+1]; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 substitution(const uint32 r_i, const uint32 q_j, const uint8 r, const uint8 q, const uint8 qq = 0) const { return q == r ? tab[2*qq] : tab[2*qq+1]; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 pattern_gap_open()            const { return pgo; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 pattern_gap_extension()       const { return pge; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 text_gap_open()               const { return tgo; }
    NVBIO_FORCEINLINE NVBIO_HOST_DEVICE int32 text_gap_extension()          const { return tge; }
};

template <uint32 BAND, aln::AlignmentType TYPE>
void run_banded_q(const TableGotohScheme scheme,
                const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                const uint8* txt, const uint32* t_off, const uint32* t_len,
                uint32 n, int32* score, uint32* sink_x, uint32* sink_y, uint8* ok)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        aln::BestSink<int32> sink;
        const bool r = aln::banded_alignment_score<BAND>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            str_view( p_len[i], qual + p_off[i] ),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            sink );
        score[i]  = sink.score; sink_x[i] = sink.sink.x; sink_y[i] = sink.sink.y;
        if (ok) ok[i] = r ? 1 : 0;
    }
}

template <aln::AlignmentType TYPE>
void run_full_q(const TableGotohScheme scheme,
              const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
              const uint8* txt, const uint32* t_off, const uint32* t_len,
              uint32 n, int32* score, uint32* sink_x, uint32* sink_y)
{
    #pragma omp parallel for schedule(dynamic,16)
    for (int64 i = 0; i < int64(n); ++i)
    {
        aln::BestSink<int32> sink;
        aln::alignment_score<4096u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            str_view( p_len[i], qual + p_off[i] ),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            sink );
        score[i]  = sink.score; sink_x[i] = sink.sink.x; sink_y[i] = sink.sink.y;
    }
}

template <uint32 BAND, aln::AlignmentType TYPE>
void run_banded(const aln::SimpleGotohScheme scheme,
                const uint8* pat, const uint32* p_off, const uint32* p_len,
                const uint8* txt, const uint32* t_off, const uint32* t_len,
                uint32 n, int32* score, uint32* sink_x, uint32* sink_y, uint8* ok)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        aln::BestSink<int32> sink;
        const bool r = aln::banded_alignment_score<BAND>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            sink );
        score[i]  = sink.score;
        sink_x[i] = sink.sink.x;
        sink_y[i] = sink.sink.y;
        if (ok) ok[i] = r ? 1 : 0;
    }
}

template <uint32 BAND>
int run_banded_type(int type, const aln::SimpleGotohScheme s,
                const uint8* pat, const uint32* p_off, const uint32* p_len,
                const uint8* txt, const uint32* t_off, const uint32* t_len,
                uint32 n, int32* score, uint32* sink_x, uint32* sink_y, uint8* ok)
{
    switch (type)
    {
    case 0: run_banded<BAND,aln::GLOBAL>     ( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0;
    case 1: run_banded<BAND,aln::LOCAL>      ( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0;
    case 2: run_banded<BAND,aln::SEMI_GLOBAL>( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0;
    }
    return -1;
}

// windowed scoring with a short2 checkpoint band (aln::banded_alignment_score<BAND>(..., window_begin, window_end, sink, checkpoint),
// nvbio/alignment/banded_inl.h:178-218): what DeviceStagedThreadScheduler runs per pass (batched_banded_inl.h:170-241)
template <uint32 BAND, aln::AlignmentType TYPE>
void run_banded_window(const aln::SimpleGotohScheme scheme,
                const uint8* pat, const uint32* p_off, const uint32* p_len,
                const uint8* txt, const uint32* t_off, const uint32* t_len,
                uint32 n, uint32 wb, uint32 we, const int32* min_score, short2* ckpt,
                int32* score, uint32* sink_x, uint32* sink_y, uint8* alive)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        if (wb == 0) { const aln::BestSink<int32> fresh; score[i] = fresh.score; sink_x[i] = fresh.sink.x; sink_y[i] = fresh.sink.y; alive[i] = 1; }   // the reference's own defaults
        if (!alive[i] || wb >= p_len[i]) continue;
        aln::BestSink<int32> sink;
        sink.score = score[i]; sink.sink = make_uint2( sink_x[i], sink_y[i] );
        const bool r = aln::banded_alignment_score<BAND>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            aln::trivial_quality_string(),
            str_view( t_len[i], txt + t_off[i] ),
            min_score ? min_score[i] : INT_MIN,
            wb, nvbio::min( we, p_len[i] ),
            sink,
            ckpt + uint64(i)*BAND );
        score[i]  = sink.score;
        sink_x[i] = sink.sink.x;
        sink_y[i] = sink.sink.y;
        alive[i]  = r ? 1 : 0;
    }
}

template <uint32 BAND>
int run_banded_window_type(int type, const aln::SimpleGotohScheme s,
                const uint8* pat, const uint32* p_off, const uint32* p_len,
                const uint8* txt, const uint32* t_off, const uint32* t_len,
                uint32 n, uint32 wb, uint32 we, const int32* min_score, short2* ckpt,
                int32* score, uint32* sink_x, uint32* sink_y, uint8* alive)
{
    switch (type)
    {
    case 0: run_banded_window<BAND,aln::GLOBAL>     ( s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,ckpt, score,sink_x,sink_y,alive ); return 0;
    case 1: run_banded_window<BAND,aln::LOCAL>      ( s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,ckpt, score,sink_x,sink_y,alive ); return 0;
    case 2: run_banded_window<BAND,aln::SEMI_GLOBAL>( s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,ckpt, score,sink_x,sink_y,alive ); return 0;
    }
    return -1;
}

// a Backtracer (nvbio/alignment/alignment.h "Backtracer" concept) that records the pushed ops (end -> start order, as
// TestBacktracker does, nvbio-test/alignment_test_utils.h:628-643) and the two clip lengths
struct RecordingBacktracer
{
    uint8* ops; uint32 n, cap; uint32 clips[2]; uint32 n_clips;
    void clip(const uint32 len) { if (n_clips < 2) clips[n_clips] = len; ++n_clips; }
    void push(const uint8 op)   { if (n < cap) ops[n] = op; ++n; }
};

template <uint32 BAND, aln::AlignmentType TYPE>
void run_traceback(const aln::SimpleGotohScheme scheme,
                   const uint8* pat, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                   uint8* ops, uint32* n_ops, uint32* clips)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        RecordingBacktracer bt; bt.ops = ops + uint64(i)*max_ops; bt.n = 0; bt.cap = max_ops; bt.n_clips = 0; bt.clips[0] = bt.clips[1] = 0;
        const aln::Alignment<int32> a = aln::banded_alignment_traceback<BAND,1024u,32u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            aln::trivial_quality_string(),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            bt );
        score[i] = a.score;
        sink_xy[2*i] = a.sink.x;     sink_xy[2*i+1] = a.sink.y;
        source_xy[2*i] = a.source.x; source_xy[2*i+1] = a.source.y;
        n_ops[i] = bt.n;
        clips[2*i] = bt.clips[0]; clips[2*i+1] = bt.clips[1];
    }
}

template <uint32 BAND>
int run_traceback_type(int type, const aln::SimpleGotohScheme s,
                   const uint8* pat, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                   uint8* ops, uint32* n_ops, uint32* clips)
{
    switch (type)
    {
    case 0: run_traceback<BAND,aln::GLOBAL>     ( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 1: run_traceback<BAND,aln::LOCAL>      ( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 2: run_traceback<BAND,aln::SEMI_GLOBAL>( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    }
    return -1;
}

template <aln::AlignmentType TYPE>
void run_full(const aln::SimpleGotohScheme scheme,
              const uint8* pat, const uint32* p_off, const uint32* p_len,
              const uint8* txt, const uint32* t_off, const uint32* t_len,
              uint32 n, int32* score, uint32* sink_x, uint32* sink_y)
{
    #pragma omp parallel for schedule(dynamic,16)
    for (int64 i = 0; i < int64(n); ++i)
    {
        aln::BestSink<int32> sink;
        aln::alignment_score<4096u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),           // default algorithm tag = PatternBlockingTag
            str_view( p_len[i], pat + p_off[i] ),
            aln::trivial_quality_string(),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            sink );
        score[i]  = sink.score;
        sink_x[i] = sink.sink.x;
        sink_y[i] = sink.sink.y;
    }
}

// full-matrix traceback through the reference's generic driver (alignment_inl.h:498-530) with its stack-allocated
// checkpoints: patterns up to 256, texts up to 512 symbols, a checkpoint every 64 pattern columns
template <aln::AlignmentType TYPE>
void run_full_traceback(const aln::SimpleGotohScheme scheme,
                   const uint8* pat, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                   uint8* ops, uint32* n_ops, uint32* clips)
{
    #pragma omp parallel for schedule(dynamic,4)
    for (int64 i = 0; i < int64(n); ++i)
    {
        RecordingBacktracer bt; bt.ops = ops + uint64(i)*max_ops; bt.n = 0; bt.cap = max_ops; bt.n_clips = 0; bt.clips[0] = bt.clips[1] = 0;
        const aln::Alignment<int32> a = aln::alignment_traceback<256u,512u,64u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            aln::trivial_quality_string(),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            bt );
        score[i] = a.score;
        sink_xy[2*i] = a.sink.x;     sink_xy[2*i+1] = a.sink.y;
        source_xy[2*i] = a.source.x; source_xy[2*i+1] = a.source.y;
        n_ops[i] = bt.n;
        clips[2*i] = bt.clips[0]; clips[2*i+1] = bt.clips[1];
    }
}

// the two tracebacks above with the table-driven scheme and the patterns' own base qualities in place of trivial_quality_string()
template <uint32 BAND, aln::AlignmentType TYPE>
void run_traceback_q(const TableGotohScheme scheme,
                   const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                   uint8* ops, uint32* n_ops, uint32* clips)
{
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        RecordingBacktracer bt; bt.ops = ops + uint64(i)*max_ops; bt.n = 0; bt.cap = max_ops; bt.n_clips = 0; bt.clips[0] = bt.clips[1] = 0;
        const aln::Alignment<int32> a = aln::banded_alignment_traceback<BAND,1024u,32u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            str_view( p_len[i], qual + p_off[i] ),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            bt );
        score[i] = a.score;
        sink_xy[2*i] = a.sink.x;     sink_xy[2*i+1] = a.sink.y;
        source_xy[2*i] = a.source.x; source_xy[2*i+1] = a.source.y;
        n_ops[i] = bt.n;
        clips[2*i] = bt.clips[0]; clips[2*i+1] = bt.clips[1];
    }
}

template <aln::AlignmentType TYPE>
void run_full_traceback_q(const TableGotohScheme scheme,
                   const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                   uint8* ops, uint32* n_ops, uint32* clips)
{
    #pragma omp parallel for schedule(dynamic,4)
    for (int64 i = 0; i < int64(n); ++i)
    {
        RecordingBacktracer bt; bt.ops = ops + uint64(i)*max_ops; bt.n = 0; bt.cap = max_ops; bt.n_clips = 0; bt.clips[0] = bt.clips[1] = 0;
        const aln::Alignment<int32> a = aln::alignment_traceback<256u,512u,64u>(
            aln::make_gotoh_aligner<TYPE>( scheme ),
            str_view( p_len[i], pat + p_off[i] ),
            str_view( p_len[i], qual + p_off[i] ),
            str_view( t_len[i], txt + t_off[i] ),
            INT_MIN,
            bt );
        score[i] = a.score;
        sink_xy[2*i] = a.sink.x;     sink_xy[2*i+1] = a.sink.y;
        source_xy[2*i] = a.source.x; source_xy[2*i+1] = a.source.y;
        n_ops[i] = bt.n;
        clips[2*i] = bt.clips[0]; clips[2*i+1] = bt.clips[1];
    }
}

} // anonymous namespace

// generic rank dictionary (SURVEY 8a row a6): the reference's rank_dictionary over a PLAIN big-endian 2-bit PackedStream of 32- or 64-bit
// words with a separate occ table every K symbols -- the two instantiations its own rank_test.cu:144-232 runs, plus other K.
// Packs `text` (n symbols), builds the table with build_occurrence_table<2,K>, answers rank(dict, i, c); words / occ are returned raw.
template <typename W, typename I, uint32 K>
static void generic_rank_impl(uint64 n, const uint8* text, W* words, I* occ, const uint64* qi, const uint8* qc, uint32 nq, uint64* out)
{
    typedef PackedStream<W*,uint8,2u,true,I>        wstream_t;
    typedef PackedStream<const W*,uint8,2u,true,I>  stream_t;
    wstream_t T( words );
    for (uint64 i = 0; i < n; ++i) T[I(i)] = text[i];
    I cnt[4];
    build_occurrence_table<2u,K>( stream_t( words ), stream_t( words ) + I(n), occ, cnt );
    uint32 ct[256]; gen_bwt_count_table( ct );
    typedef rank_dictionary<2u,K,stream_t,const I*,const uint32*> dict_t;
    const dict_t dict( stream_t( words ), occ, ct );
    for (uint32 q = 0; q < nq; ++q)
        out[q] = uint64( rank( dict, qi[q] == ~uint64(0) ? I(-1) : I(qi[q]), uint32( qc[q] ) ) );
}

extern "C" {

// full-matrix Gotoh traceback: aln::alignment_traceback<256,512,64> (nvbio/alignment/alignment_inl.h:365-530)
int ref_gotoh_full_traceback(int type, int match, int mismatch, int gap_open, int gap_ext,
                     const uint8* pat, const uint32* p_off, const uint32* p_len,
                     const uint8* txt, const uint32* t_off, const uint32* t_len,
                     uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                     uint8* ops, uint32* n_ops, uint32* clips)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    for (uint32 i = 0; i < n; ++i) if (p_len[i] > 256u || t_len[i] > 512u) return -2;
    switch (type)
    {
    case 0: run_full_traceback<aln::GLOBAL>     ( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 1: run_full_traceback<aln::LOCAL>      ( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 2: run_full_traceback<aln::SEMI_GLOBAL>( s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    }
    return -1;
}

// full-matrix Gotoh score: aln::alignment_score<MAX_TEXT_LEN>(GotohAligner<TYPE,SimpleGotohScheme>, ...)
// (nvbio/alignment/alignment_inl.h:95-125 -> gotoh/gotoh_inl.h:459-960, PatternBlockingTag); texts up to 4096 symbols
int ref_gotoh_full(int type, int match, int mismatch, int gap_open, int gap_ext,
                   const uint8* pat, const uint32* p_off, const uint32* p_len,
                   const uint8* txt, const uint32* t_off, const uint32* t_len,
                   uint32 n, int32* score, uint32* sink_x, uint32* sink_y)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    switch (type)
    {
    case 0: run_full<aln::GLOBAL>     ( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    case 1: run_full<aln::LOCAL>      ( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    case 2: run_full<aln::SEMI_GLOBAL>( s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    }
    return -1;
}

// banded Gotoh traceback (aln::banded_alignment_traceback<BAND,1024,32>, nvbio/alignment/banded_inl.h:352-489):
// ops are the backtracer's pushes in END -> START order (0 = SUBSTITUTION 'M', 1 = INSERTION 'I', 2 = DELETION 'D'),
// clips = (pattern_len - sink.y, source.y)
int ref_banded_traceback(int band, int type, int match, int mismatch, int gap_open, int gap_ext,
                     const uint8* pat, const uint32* p_off, const uint32* p_len,
                     const uint8* txt, const uint32* t_off, const uint32* t_len,
                     uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                     uint8* ops, uint32* n_ops, uint32* clips)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    switch (band)
    {
    case  7: return run_traceback_type< 7>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips );
    case 15: return run_traceback_type<15>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips );
    case 31: return run_traceback_type<31>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips );
    }
    return -1;
}


int ref_num_threads() { return omp_get_max_threads(); }
void ref_set_num_threads(int t) { omp_set_num_threads(t); }

// text: n unpacked symbols in {0..3}.  Outputs: sa[n+1] (sa[0]=n), bwt words (2-bit big-endian,
// `bwt_words` uint32 words, caller-zeroed), returns primary.
uint32 ref_build_bwt(uint32 n, const uint8* text, int32* sa, uint32* bwt, uint32 bwt_words)
{
    std::vector<uint32> twords( (n + 15)/16 + 4, 0u );
    typedef PackedStream<uint32*,uint8,2u,true> stream_t;
    stream_t T( &twords[0] );
    for (uint32 i = 0; i < n; ++i) T[i] = text[i];

    gen_sa( n, T, sa );
    std::memset( bwt, 0, sizeof(uint32)*bwt_words );
    stream_t B( bwt );
    return gen_bwt_from_sa( n, T, sa, B );
}

// occ: ceil(n/64)*4 words; cnt: 4 words
void ref_build_occ(uint32 n, const uint32* bwt, uint32* occ, uint32* cnt)
{
    typedef PackedStream<const uint32*,uint8,2u,true> stream_t;
    stream_t B( bwt );
    build_occurrence_table<2u,64u>( B, B + n, occ, cnt );
}

void ref_count_table(uint32* table) { gen_bwt_count_table( table ); }

// ssa[(n+16)/16] from a full SA (sa[0] = n), then ssa[0] = -1 as the loader does
// (nvbio/io/fmindex/fmindex_impl.cu:244)
void ref_build_ssa(uint32 n, const int32* sa, uint32* ssa)
{
    SSA_index_multiple<16u> s( n, (const uint32*)sa );
    const uint32 n_items = (n + 16u)/16u;
    for (uint32 i = 0; i < n_items; ++i) ssa[i] = s.m_ssa[i];
    ssa[0] = uint32(-1);
}

// rank(fmi, k, c) for many (k,c)
void ref_rank(const uint32* bwt_occ, const uint32* L2, uint32 n, uint32 primary,
              const uint32* k, const uint8* c, uint32 nq, uint32* out)
{
    uint32 ct[256]; gen_bwt_count_table( ct );
    const fm_index_t fmi = make_index( bwt_occ, NULL, L2, ct, n, primary );
    for (uint32 i = 0; i < nq; ++i) out[i] = rank( fmi, k[i], c[i] );
}

// dictionary-level rank over the interleaved layout (no $ correction): rank(dict, i, c)
void ref_dict_rank(const uint32* bwt_occ, const uint32* idx, const uint8* c, uint32 nq, uint32* out)
{
    uint32 ct[256]; gen_bwt_count_table( ct );
    const bwt_occ_ptr p = (const uint4*)bwt_occ;
    const rank_dict_t dict( bwt_stream( bwt_iter(p) ), occ_iter(p), ct );
    for (uint32 i = 0; i < nq; ++i) out[i] = rank( dict, idx[i], uint32(c[i]) );
}

// match(): queries are unpacked symbols, query i = q[off[i] .. off[i]+len[i]); out = inclusive (x,y)
void ref_match(const uint32* bwt_occ, const uint32* L2, uint32 n, uint32 primary,
               const uint8* q, const uint32* off, const uint32* len, uint32 nq, uint32* out_xy)
{
    uint32 ct[256]; gen_bwt_count_table( ct );
    const fm_index_t fmi = make_index( bwt_occ, NULL, L2, ct, n, primary );
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(nq); ++i)
    {
        const uint2 r = match( fmi, q + off[i], len[i] );
        out_xy[2*i+0] = r.x;
        out_xy[2*i+1] = r.y;
    }
}

// locate(): SA rows -> text positions
void ref_locate(const uint32* bwt_occ, const uint32* ssa, const uint32* L2, uint32 n, uint32 primary,
                const uint32* rows, uint32 nq, uint32* out)
{
    uint32 ct[256]; gen_bwt_count_table( ct );
    const fm_index_t fmi = make_index( bwt_occ, ssa, L2, ct, n, primary );
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(nq); ++i)
        out[i] = locate( fmi, rows[i] );
}

// banded Gotoh score with SimpleGotohScheme(match, mismatch, gap_open, gap_ext).
// type: 0 GLOBAL, 1 LOCAL, 2 SEMI_GLOBAL (nvbio/alignment/alignment_base.h:54)
// quality-table scheme (6 gap/none constants come as scheme6 = {unused, unused, pgo, pge, tgo, tge}) through the same templates
int ref_banded_gotoh_q(int band, int type, const int32* scheme6, const int32* qtab,
                       const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                       const uint8* txt, const uint32* t_off, const uint32* t_len,
                       uint32 n, int32* score, uint32* sink_x, uint32* sink_y, uint8* ok)
{
    TableGotohScheme s; s.tab = qtab; s.pgo = scheme6[2]; s.pge = scheme6[3]; s.tgo = scheme6[4]; s.tge = scheme6[5];
#define REF_BQ(B) switch (type) { \
    case 0: run_banded_q<B,aln::GLOBAL>     ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0; \
    case 1: run_banded_q<B,aln::LOCAL>      ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0; \
    case 2: run_banded_q<B,aln::SEMI_GLOBAL>( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok ); return 0; } return -1;
    switch (band) { case 7: REF_BQ(7) case 15: REF_BQ(15) case 31: REF_BQ(31) }
#undef REF_BQ
    return -1;
}

int ref_gotoh_full_q(int type, const int32* scheme6, const int32* qtab,
                     const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                     const uint8* txt, const uint32* t_off, const uint32* t_len,
                     uint32 n, int32* score, uint32* sink_x, uint32* sink_y)
{
    TableGotohScheme s; s.tab = qtab; s.pgo = scheme6[2]; s.pge = scheme6[3]; s.tgo = scheme6[4]; s.tge = scheme6[5];
    switch (type)
    {
    case 0: run_full_q<aln::GLOBAL>     ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    case 1: run_full_q<aln::LOCAL>      ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    case 2: run_full_q<aln::SEMI_GLOBAL>( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y ); return 0;
    }
    return -1;
}

// quality-table tracebacks (scheme6 = {unused, unused, pgo, pge, tgo, tge}): the banded one at every band ref_banded_gotoh_q
// instantiates, the full-matrix one with patterns up to 256 and texts up to 512 symbols
int ref_banded_traceback_q(int band, int type, const int32* scheme6, const int32* qtab,
                           const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                           const uint8* txt, const uint32* t_off, const uint32* t_len,
                           uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                           uint8* ops, uint32* n_ops, uint32* clips)
{
    TableGotohScheme s; s.tab = qtab; s.pgo = scheme6[2]; s.pge = scheme6[3]; s.tgo = scheme6[4]; s.tge = scheme6[5];
#define REF_TQ(B) switch (type) { \
    case 0: run_traceback_q<B,aln::GLOBAL>     ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0; \
    case 1: run_traceback_q<B,aln::LOCAL>      ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0; \
    case 2: run_traceback_q<B,aln::SEMI_GLOBAL>( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0; } return -1;
    switch (band) { case 7: REF_TQ(7) case 15: REF_TQ(15) case 31: REF_TQ(31) }
#undef REF_TQ
    return -1;
}

int ref_gotoh_full_traceback_q(int type, const int32* scheme6, const int32* qtab,
                               const uint8* pat, const uint8* qual, const uint32* p_off, const uint32* p_len,
                               const uint8* txt, const uint32* t_off, const uint32* t_len,
                               uint32 n, uint32 max_ops, int32* score, uint32* sink_xy, uint32* source_xy,
                               uint8* ops, uint32* n_ops, uint32* clips)
{
    TableGotohScheme s; s.tab = qtab; s.pgo = scheme6[2]; s.pge = scheme6[3]; s.tgo = scheme6[4]; s.tge = scheme6[5];
    for (uint32 i = 0; i < n; ++i) if (p_len[i] > 256u || t_len[i] > 512u) return -2;
    switch (type)
    {
    case 0: run_full_traceback_q<aln::GLOBAL>     ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 1: run_full_traceback_q<aln::LOCAL>      ( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    case 2: run_full_traceback_q<aln::SEMI_GLOBAL>( s, pat,qual,p_off,p_len, txt,t_off,t_len, n, max_ops, score,sink_xy,source_xy,ops,n_ops,clips ); return 0;
    }
    return -1;
}

int ref_banded_gotoh_window(int band, int type, int match, int mismatch, int gap_open, int gap_ext,
                     const uint8* pat, const uint32* p_off, const uint32* p_len,
                     const uint8* txt, const uint32* t_off, const uint32* t_len,
                     uint32 n, uint32 wb, uint32 we, const int32* min_score, short* ckpt,
                     int32* score, uint32* sink_x, uint32* sink_y, uint8* alive)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    switch (band)
    {
    case  7: return run_banded_window_type< 7>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,(short2*)ckpt, score,sink_x,sink_y,alive );
    case 15: return run_banded_window_type<15>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,(short2*)ckpt, score,sink_x,sink_y,alive );
    case 31: return run_banded_window_type<31>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, wb,we,min_score,(short2*)ckpt, score,sink_x,sink_y,alive );
    }
    return -1;
}

int ref_banded_gotoh(int band, int type, int match, int mismatch, int gap_open, int gap_ext,
                     const uint8* pat, const uint32* p_off, const uint32* p_len,
                     const uint8* txt, const uint32* t_off, const uint32* t_len,
                     uint32 n, int32* score, uint32* sink_x, uint32* sink_y, uint8* ok)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    switch (band)
    {
    case  3: return run_banded_type< 3>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    case  5: return run_banded_type< 5>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    case  7: return run_banded_type< 7>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    case 15: return run_banded_type<15>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    case 31: return run_banded_type<31>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    case 63: return run_banded_type<63>( type, s, pat,p_off,p_len, txt,t_off,t_len, n, score,sink_x,sink_y,ok );
    }
    return -1;
}


int ref_generic_rank(int word_bits, uint32 K, uint64 n, const uint8* text, void* words, void* occ, const uint64* qi, const uint8* qc, uint32 nq, uint64* out)
{
    if (word_bits == 32 && K == 64)  { generic_rank_impl<uint32,uint32,64> ( n, text, (uint32*)words, (uint32*)occ, qi, qc, nq, out ); return 0; }
    if (word_bits == 32 && K == 128) { generic_rank_impl<uint32,uint32,128>( n, text, (uint32*)words, (uint32*)occ, qi, qc, nq, out ); return 0; }
    if (word_bits == 32 && K == 16)  { generic_rank_impl<uint32,uint32,16> ( n, text, (uint32*)words, (uint32*)occ, qi, qc, nq, out ); return 0; }
    if (word_bits == 64 && K == 64)  { generic_rank_impl<uint64,uint64,64> ( n, text, (uint64*)words, (uint64*)occ, qi, qc, nq, out ); return 0; }
    if (word_bits == 64 && K == 256) { generic_rank_impl<uint64,uint64,256>( n, text, (uint64*)words, (uint64*)occ, qi, qc, nq, out ); return 0; }
    return -1;
}


// banded Gotoh with aln::Best2Sink<int32>(distinct_dist) (nvbio/alignment/sink.h:114-147): out6 = (score1, sink1, score2, sink2) per alignment
int ref_banded_gotoh_best2(int band, int type, int match, int mismatch, int gap_open, int gap_ext,
                           const uint8* pat, const uint32* p_off, const uint32* p_len, const uint8* txt, const uint32* t_off, const uint32* t_len,
                           uint32 n, uint32 distinct_dist, long long* out6)
{
    const aln::SimpleGotohScheme s( match, mismatch, gap_open, gap_ext );
    #pragma omp parallel for schedule(static)
    for (int64 i = 0; i < int64(n); ++i)
    {
        aln::Best2Sink<int32> sink( distinct_dist );
        const str_view P( p_len[i], pat + p_off[i] ), T( t_len[i], txt + t_off[i] );
#define B2(B, TY) aln::banded_alignment_score<B>( aln::make_gotoh_aligner<TY>( s ), P, T, INT_MIN, sink )
        if (band == 15) { if (type == 0) B2(15, aln::GLOBAL); else if (type == 1) B2(15, aln::LOCAL); else B2(15, aln::SEMI_GLOBAL); }
        else if (band == 31) { if (type == 0) B2(31, aln::GLOBAL); else if (type == 1) B2(31, aln::LOCAL); else B2(31, aln::SEMI_GLOBAL); }
        else { if (type == 0) B2(7, aln::GLOBAL); else if (type == 1) B2(7, aln::LOCAL); else B2(7, aln::SEMI_GLOBAL); }
#undef B2
        long long* o = out6 + 6 * i;
        o[0] = sink.score1; o[1] = sink.sink1.x; o[2] = sink.sink1.y; o[3] = sink.score2; o[4] = sink.sink2.x; o[5] = sink.sink2.y;
    }
    return (band == 7 || band == 15 || band == 31) ? 0 : -1;
}

} // extern "C"
