/* nvbio_b200.h -- C ABI of the H100-native replacement for nvbio's two data-parallel hot paths.
 *
 * Plain C: pointers, sizes, PODs.  No torch / thrust / nvbio types in any signature.
 * All `d_` pointers are DEVICE memory owned by the caller; all calls are asynchronous on `stream`
 * (a cudaStream_t passed as void*; NULL = the legacy default stream) unless stated otherwise.
 * Return value: 0 on success, a positive cudaError_t value, or a negative NVB_E_* code.
 *
 * Every entry point names the reference interface it replaces (paths relative to the nvbio tree).
 * INTEGRATION.md shows the reference-side binding for each.
 *
 * Threads and devices.  Every call works on the CURRENT device of the calling thread (cudaSetDevice), and all `d_` pointers must
 * belong to it.  The library keeps no state between calls except, per device, lazily-created profiling events and kernel
 * attributes (both guarded; a host that drives several GPUs from one process -- nvBowtie's one compute thread per device -- may
 * call from all of its threads at once).  Two concurrent calls must not share output or temp buffers.
 */
#ifndef NVBIO_B200_H
#define NVBIO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NVB_VERSION 100

/* error codes (negative; positive values are cudaError_t) */
#define NVB_OK              0
#define NVB_E_INVALID      -1   /* bad argument (unsupported band length, bits, NULL pointer, ...) */
#define NVB_E_TEMP_SIZE    -2   /* temp buffer too small: *temp_bytes holds the required size */
#define NVB_E_CAPACITY     -3   /* an output buffer capacity would be exceeded */
#define NVB_E_UNSUPPORTED  -4   /* valid request that this build does not implement */

typedef struct nvb_uint2 { uint32_t x, y; } nvb_uint2;

/* score of an alignment sink that received no report: nvbio's Field_traits<int32>::min() (nvbio/basic/numbers.h:832-836), the value
 * aln::BestSink<int32> / Best2Sink<int32> are constructed with (sink_inl.h:40,73-78) */
#define NVB_SINK_MIN (-(1 << 30))

/* ---------------------------------------------------------------------------------------------
 * Data views
 * ------------------------------------------------------------------------------------------- */

/* FM-index in the reference's production layout (nvbio/io/fmindex/fmindex.h:302-319,
 * nvbio/io/fmindex/fmindex_impl.cu:308-322): block k = 32 bytes at byte offset 32k =
 * { uint4 bwt = 64 symbols, 2-bit big-endian ; uint4 occ = #A,#C,#G,#T in bwt[0,64k) }.
 * Mirrors nvbio::fm_index<rank_dictionary<2,64,...>, SSA_index_multiple_context<16>>
 * (nvbio/fmindex/fmindex.h:341-387): {m_length, m_primary, m_L2, m_rank_dict, m_sa}. */
/* The longest text an index may have: the empty query's range (0, n) has 1 + n rows, which must fit a uint32 range size. */
#define NVB_FM_MAX_LENGTH  0xFFFFFFFEu

typedef struct nvb_fm_index {
    const void*     d_bwt_occ;   /* ceil(length/64) blocks of 32 bytes, 32-byte aligned            */
    const uint32_t* d_ssa;       /* (length+I)/I words: SA[r] for r%I==0, ssa[0]=0xFFFFFFFF; may be
                                    NULL when only rank/match are used                             */
    uint32_t        length;      /* text length n (number of BWT symbols), at most NVB_FM_MAX_LENGTH   */
    uint32_t        primary;     /* row of the `$` suffix                                          */
    uint32_t        L2[5];       /* exclusive prefix sums of the symbol counts                     */
    /* ---- optional extensions; zero-initialise for an index in the reference's format ---- */
    uint32_t        sa_interval; /* I: 0 or 16 = the reference's SA_INT (FMIndexDataCore::SA_INT);
                                    any power of two down to 1 (= the full suffix array, 4 bytes per
                                    base: 7.6 GB at 1.9 Gbp, affordable on an 80 GB part) shortens locate  */
    const nvb_uint2* d_ktab;     /* 4^ktab_k inclusive SA ranges of every k-mer (index = the k symbols
                                    as a 2k-bit number, first symbol most significant), built by
                                    nvb_fm_build_ktab; replaces the first k LF steps of match()     */
    uint32_t        ktab_k;      /* 0 = no table */
    uint32_t        ktab_located;/* 0: d_ktab holds 8-byte entries {x, y};  1: 16-byte entries {x, y, SA[x], SA[y]} built by
                                    nvb_fm_build_ktab_located (SA[x] valid when y == x, both when y == x + 1): a seed whose
                                    k-mer occurs once or twice is located by the look-up + a text comparison, without walking the
                                    range on;  2: the same table built by nvb_fm_build_ktab_context -- the last word of a ONE-row
                                    entry (y == x) holds the 16 text symbols before SA[x] instead, so that such a seed (up to k + 16
                                    symbols long) is resolved by the look-up alone; and, when length < 0xC0000000, a TWO-row entry is
                                    stored as {x, 0xC0000000 | a | b << 14, SA[x], SA[x+1]} (y = x + 1 implied; a, b = the 7 symbols before
                                    SA[x], SA[x+1]), which resolves seeds up to k + 7 symbols the same way;  3: as 2, and d_rows is set
                                    (needs sa_interval == 1 and d_ssa);  4: d_ktab holds 32-byte entries (32-byte aligned) built by
                                    nvb_fm_build_ktab_wide: the first 16 bytes of each as at level 2, and a k-mer with 3 to 8
                                    occurrences also carries its rows' text contexts (and, for 3 or 4 rows, their SA values), so that
                                    the seed + extend path resolves most such seeds with the look-up alone (needs sa_interval == 1 and
                                    d_ssa);  5: as 4, and d_rows is set.  Ranges are identical in every case.  */
    const nvb_uint2* d_rows;     /* read only when ktab_located is 3 or 5: length + 1 entries {SA[r], the 16 text symbols before SA[r]}
                                    built by nvb_fm_build_rows.  The per-read seed + extend path then resolves a seed whose k-mer
                                    occurs 3 to 8 times (and that is up to k + 16 symbols long) with one gather of those rows instead
                                    of walking the range on; results are identical with and without it */
} nvb_fm_index;

/* A set of strings stored in one packed symbol stream (nvbio PackedStream semantics,
 * nvbio/basic/packedstream_inl.h:336-372): `bits` per symbol in {2,4,8}; big_endian = symbol 0 of a
 * word sits in its TOP bits (nvbio's BIG_ENDIAN_T).  String i spans symbols
 * [off_i, off_i+len_i) of the stream, with
 *     off_i = d_offsets ? d_offsets[i] : i * stride,   len_i = d_lengths ? d_lengths[i] : length.
 * This covers ConcatenatedStringSet / SparseStringSet / fixed-stride sets over a packed stream
 * (nvbio/strings/string_set.h) and the infix sets built by extract_seeds (nvbio/strings/seeds.h).  Strings may share or overlap
 * symbols, and offsets use the whole uint32 range: off_i + len_i may reach 2^32. */
typedef struct nvb_string_set {
    const uint32_t* d_words;
    uint32_t        bits;
    uint32_t        big_endian;
    const uint32_t* d_offsets;
    const uint32_t* d_lengths;
    uint32_t        stride;
    uint32_t        length;
} nvb_string_set;

/* alignment type, values of nvbio::aln::AlignmentType (nvbio/alignment/alignment_base.h:54) */
#define NVB_GLOBAL      0
#define NVB_LOCAL       1
#define NVB_SEMI_GLOBAL 2

/* Gotoh scoring scheme.  With d_qual_table == NULL this is aln::SimpleGotohScheme
 * (nvbio/alignment/utils.h:114-135: substitution = r==q ? match : mismatch).  With a table it is
 * nvBowtie's SmithWatermanScoringScheme<QualCost,ConstantCost>::substitution
 * (nvBowtie/bowtie2/cuda/scoring.h:281): r==q ? table[2*qual] : table[2*qual+1]; the caller evaluates
 * the reference's float expression (scoring.h:96-100) on the host into the 256x2 int32 table so that
 * fast-math differences cannot leak in.  All gap costs are negative. */
typedef struct nvb_gotoh_scheme {
    int32_t        match, mismatch;
    int32_t        pattern_gap_open, pattern_gap_ext;
    int32_t        text_gap_open, text_gap_ext;
    const int32_t* d_qual_table;     /* device, 512 int32, or NULL */
    int32_t        qual_table_min;   /* bounds of the table's values (host knowledge of device data): they admit the */
    int32_t        qual_table_max;   /* packed 16-bit DPX path; 0,0 = unknown -> the int32 kernel scores the batch   */
} nvb_gotoh_scheme;

int         nvb_version(void);
const char* nvb_error_string(int err);

/* ---------------------------------------------------------------------------------------------
 * HP-A  FM-index
 * ------------------------------------------------------------------------------------------- */

/* out[i] = rank(fmi, k[i], c[i]) : occurrences of c in bwt rows [0,k], `$`-aware.
 * Replaces nvbio::rank(fm_index,k,c)  (nvbio/fmindex/fmindex_inl.h:36-57 ->
 * rank_dictionary_inl.h:500-511 dispatch_rank<2,64,...,uint4,uint4>::run). */
int nvb_fm_rank(const nvb_fm_index* fmi, const uint32_t* d_k, const uint8_t* d_c, uint32_t n,
                uint32_t* d_out, void* stream);

/* d_out4[4*i + c] = rank(fmi, k[i], c) for c = A,C,G,T at once (16-byte aligned output).
 * Replaces nvbio::rank4(fm_index,k) / rank_all (nvbio/fmindex/fmindex_inl.h:107-133,194-222 ->
 * rank_dictionary_inl.h:539-573, the count-table popc_2bit_all path used by nvBowtie's 1-mismatch mapper). */
int nvb_fm_rank4(const nvb_fm_index* fmi, const uint32_t* d_k, uint32_t n, uint32_t* d_out4, void* stream);

/* Generic rank dictionary (SURVEY 8a row a6): a PLAIN big-endian 2-bit packed text over 32- or 64-bit words with a separate
 * occurrence table sampled every K symbols (K a multiple of the symbols per word), 32- or 64-bit counters -- the form the
 * reference's tests and its 64-bit indices instantiate.  Replaces dispatch_rank<2,K,PackedStream<...,2,true,index_type>,Occ,CT,
 * word_type,index_type>::run / run4 (nvbio/fmindex/rank_dictionary_inl.h:243-422) and build_occurrence_table<2,K> (:42-77).
 *   d_occ[4k + c]    = #c in text[0, kK)          (index_bits wide)
 *   nvb_dict_rank    d_out[t] = #c[t] in text[0, i[t]]  (i and out index_bits wide; i == all ones -> 0)
 *   nvb_dict_rank4   d_out4[4t + c] for c = A,C,G,T
 *   nvb_dict_build_occ  builds d_occ (ceil(n/K) * 4 counters) on the device; h_counts (optional) = the four symbol totals */
int nvb_dict_rank(const void* d_text, uint32_t word_bits, const void* d_occ, uint32_t index_bits, uint32_t K,
                  const void* d_i, const uint8_t* d_c, uint32_t n, void* d_out, void* stream);
int nvb_dict_rank4(const void* d_text, uint32_t word_bits, const void* d_occ, uint32_t index_bits, uint32_t K,
                   const void* d_i, uint32_t n, void* d_out4, void* stream);
int nvb_dict_build_occ(const void* d_text, uint32_t word_bits, uint64_t n_symbols, uint32_t K, uint32_t index_bits, void* d_occ, uint64_t h_counts[4],
                       void* d_temp, size_t* temp_bytes, void* stream);

#define NVB_MATCH_FORWARD_ORDER 1u  /* consume the query left-to-right instead of right-to-left   */
#define NVB_MATCH_COMPLEMENT    2u  /* complement each symbol (c<4 ? 3-c : c) before ranking      */
/* FORWARD_ORDER|COMPLEMENT is how nvBowtie searches the reverse-complement strand of a seed over the
 * forward index (nvBowtie/bowtie2/cuda/mapping_inl.h:292-309). */

/* Exact backward search of n queries: d_ranges[i] = inclusive SA range (x,y), empty iff x>y;
 * a query symbol > 3 yields (1,0).
 * Replaces nvbio::match(fm_index,pattern,len) (nvbio/fmindex/fmindex_inl.h:280-341), nvBowtie's
 * match_range (nvBowtie/bowtie2/cuda/mapping_inl.h:83-97) and the thrust::transform(rank_functor) of
 * FMIndexFilter::rank (nvbio/fmindex/filter_inl.h:283-287). */
int nvb_fm_match(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                 nvb_uint2* d_ranges, void* stream);

/* One-mismatch seed search: nvBowtie's map<find_exact>(query, len1, len2, index, ...) as a batch primitive
 * (nvBowtie/bowtie2/cuda/mapping_inl.h:128-220, the rank4-based core of the APPROX / CASE_PRUNING seed mappers,
 * :318-429).  For query i: every SA range of the query with exactly one substitution among its consumed symbols
 * [exact_len, len) (none in the first exact_len), in the reference's push order (position ascending, substituted
 * symbol ascending), followed by the perfect match when find_exact; an N inside the exact region or a second N yields
 * nothing, a single later N ends exact matching there.  "Consumed symbols" are the stream's symbols in order with
 * NVB_MATCH_FORWARD_ORDER (nvBowtie's forward reader over its reversed reads), reversed without it.
 * d_ranges[i*max_out + k] = k-th inclusive range (k < min(count, max_out)); d_counts[i] = pushes; d_range_sums[i]
 * (optional) = sum of the range sizes (the reference's range_sum; range_count = count).
 * The bounded priority deque the reference feeds (seed_hit_deque_array.h) stays with the caller. */
int nvb_fm_match_approx(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                        uint32_t exact_len, int find_exact, uint32_t max_out,
                        nvb_uint2* d_ranges, uint32_t* d_counts, uint32_t* d_range_sums, void* stream);

/* -------------------------------------------------------------------------------------------
 * nvBowtie's seed-mapping stage (SURVEY 8a row a10 / 8f-2): for every queued read, the seeds at symbol offsets
 *     begin + retry * (seed_freq / (max_reseed + 1)) + k * seed_freq      while the seed fits
 * are searched on both strands -- exactly (EXACT) or with one substitution outside the first subseed_len consumed symbols
 * (APPROX) -- and their SA ranges kept in a BOUNDED per-read priority deque of at most max_hits SeedHits ordered by range
 * size.  Replaces map_queues_kernel<EXACT_MAPPING|APPROX_MAPPING> (nvBowtie/bowtie2/cuda/mapping_inl.h:229-366, 539-591),
 * the entry points map / map_exact / map_approx (mapping.cu:63-188) and the deque storage (seed_hit_deque_array.h:157-204).
 * CASE_PRUNING mapping needs the reverse index and is not implemented.
 *   reads            big-endian strings of 4-bit (DNA_N) or 2-bit symbols (little-endian ones are NVB_E_UNSUPPORTED); nvBowtie
 *                    reads the forward strand of a seed front to back (NVB_MATCH_FORWARD_ORDER) and the other strand back to
 *                    front, complemented (mapping_inl.h:263-309)
 *                    A seed containing an N is skipped by both mappers (as the reference's N test does, mapping_inl.h:258,346).
 *   d_queue          read ids to process (PingPongQueuesView::in_queue), or NULL = 0 .. n_queue-1
 *   d_seed_freq      optional per-read seed interval (nvBowtie evaluates SimpleFunc(read length) in float on the device,
 *                    params.cpp:157-158: evaluate it on the host); NULL = params->seed_freq for every read
 *   d_hits           arena of max_hits slots per READ ID: the read's hits sorted by range size (ascending, stable in push
 *                    order = the order pop_top() yields); d_counts[read id] = their number
 *   d_reseed[i]      (optional) 1 when queue entry i found no range or range_sum >= rep_seeds * range_count (:586-588)
 *   d_range_stats    (optional) [2*i] = range_sum, [2*i+1] = range_count of queue entry i
 * A full deque drops a largest range before every further push, as the reference does (pop_bottom, then push); among equally
 * large ranges the most recently pushed one goes (an interval heap's choice depends on its layout): the kept range SIZES, the
 * statistics and -- whenever a read pushes at most max_hits hits -- the complete hit sets equal the reference's. */
typedef struct nvb_seed_hit {          /* bowtie2::cuda::SeedHit, seed_hit.h:54-98,230-232 (8 bytes) */
    uint32_t range_begin;              /* SA range [range_begin, range_begin + delta) -- EXCLUSIVE end */
    uint32_t bits;                     /* delta:20 | pos_in_read:10 | rc:1 | index_dir:1 (low to high) */
} nvb_seed_hit;
#define NVB_MAP_EXACT  0u
#define NVB_MAP_APPROX 1u
#define NVB_MAP_MAX_PUSHES 100u        /* an approximate seed of length L pushes at most 3 L + 1 ranges: L <= 33 */
typedef struct nvb_map_params {
    uint32_t algorithm;                /* NVB_MAP_EXACT | NVB_MAP_APPROX */
    uint32_t seed_len, seed_freq;      /* ParamsPOD::seed_len, seed_freq(read_len) evaluated on the host */
    uint32_t max_hits, max_reseed, rep_seeds, subseed_len, min_read_len;
    uint32_t fw, rc;                   /* search the forward / the reverse-complement strand */
} nvb_map_params;
int nvb_map_seeds(const nvb_fm_index* fmi, const nvb_string_set* reads, const uint32_t* d_queue, uint32_t n_queue, uint32_t retry,
                  const nvb_map_params* params, const uint32_t* d_seed_freq,
                  nvb_seed_hit* d_hits, uint32_t* d_counts, uint8_t* d_reseed, uint32_t* d_range_stats, void* stream);

/* Two-phase locate of queued SA rows (nvBowtie/bowtie2/cuda/locate_inl.h:122-210; nvbio/fmindex/fmindex_inl.h:502-569
 * locate_ssa_iterator / lookup_ssa_iterator): init walks LF to the next sampled row, lookup adds the sampled position.
 * d_idx (optional) is the sorting permutation nvBowtie passes as idx_queue: entry t works on element d_idx[t] of the arrays. */
int nvb_fm_locate_init(const nvb_fm_index* fmi, const uint32_t* d_rows, const uint32_t* d_idx, uint32_t n,
                       uint32_t* d_sampled_row, uint32_t* d_steps, void* stream);
int nvb_fm_locate_lookup(const nvb_fm_index* fmi, const uint32_t* d_sampled_row, const uint32_t* d_steps, const uint32_t* d_idx, uint32_t n,
                         uint32_t* d_pos, void* stream);
/* locate with the rows radix-sorted first "to gather locality" (aligner_best_approx.h:737-756): same positions as nvb_fm_locate,
 * returned in the input order. */
int nvb_fm_locate_sorted(const nvb_fm_index* fmi, const uint32_t* d_rows, uint32_t n, uint32_t* d_pos,
                         void* d_temp, size_t* temp_bytes, void* stream);

/* d_pos[i] = text position of SA row d_rows[i]  (row 0 -> 0xFFFFFFFF as in the reference).
 * Replaces nvbio::locate(fm_index,i) (nvbio/fmindex/fmindex_inl.h:471-499) with
 * SSA_index_multiple_context<16>::fetch (nvbio/fmindex/ssa_inl.h:487-504). */
int nvb_fm_locate(const nvb_fm_index* fmi, const uint32_t* d_rows, uint32_t n, uint32_t* d_pos, void* stream);

/* FMIndexFilter<device_tag>::rank (nvbio/fmindex/filter_inl.h:268-300): match every query, then
 * d_slots = inclusive scan of the range sizes (uint64).  The total hit count is d_slots[n-1]; if
 * h_n_hits != NULL the call synchronises the stream and stores it there (the reference returns it). */
int nvb_fm_filter_rank(const nvb_fm_index* fmi, const nvb_string_set* queries, uint32_t n, uint32_t flags,
                       nvb_uint2* d_ranges, uint64_t* d_slots, uint64_t* h_n_hits,
                       void* d_temp, size_t* temp_bytes, void* stream);

/* FMIndexFilter<device_tag>::locate(begin,end,hits) (nvbio/fmindex/filter_inl.h:306-402):
 * for global hit index h in [begin,end): d_hits[h-begin] = (text position, query id). */
int nvb_fm_filter_locate(const nvb_fm_index* fmi, const nvb_uint2* d_ranges, const uint64_t* d_slots,
                         uint32_t n_queries, uint64_t begin, uint64_t end, nvb_uint2* d_hits, void* stream);

/* ---------------------------------------------------------------------------------------------
 * HP-B  batched banded Gotoh score
 * ------------------------------------------------------------------------------------------- */

/* For i < n: banded DP of patterns[i] (rows) against texts[i] (band anchored at text offset 0),
 * d_score[i] / d_sink[i] = BestSink<int32>{score, sink=(text_end, pattern_end)}; an alignment with
 * text_len < pattern_len leaves the sink at its defaults (NVB_SINK_MIN, (-1,-1)).
 * band_len in {3,5,7,15,31,63}.  d_quals (one byte per pattern symbol, indexed like the pattern
 * stream) may be NULL (trivial_quality_string).
 * Replaces aln::BatchedBandedAlignmentScore<BAND_LEN,stream,DeviceThreadScheduler>::enact and
 * aln::batch_banded_alignment_score<BAND_LEN> with GotohAligner (nvbio/alignment/batched_banded_inl.h:
 * 78-162, nvbio/alignment/batched_inl.h:1067-1101 -> gotoh/gotoh_banded_inl.h:406-658).
 * Temp storage follows the reference's min_temp_storage/enact(temp_size,temp) convention
 * (nvbio/alignment/batched.h:333-353): call with d_temp==NULL to query *temp_bytes. */
int nvb_banded_gotoh_score(int band_len, int type, const nvb_gotoh_scheme* scheme,
                           const nvb_string_set* patterns, const uint8_t* d_quals,
                           const nvb_string_set* texts, uint32_t n,
                           int32_t* d_score, nvb_uint2* d_sink,
                           void* d_temp, size_t* temp_bytes, void* stream);

/* same, reading the number of alignments from device memory (*d_n <= n_max): lets a pipeline chain
 * locate -> extend without a host round trip. */
int nvb_banded_gotoh_score_indirect(int band_len, int type, const nvb_gotoh_scheme* scheme,
                           const nvb_string_set* patterns, const uint8_t* d_quals,
                           const nvb_string_set* texts, const uint32_t* d_n, uint32_t n_max,
                           int32_t* d_score, nvb_uint2* d_sink,
                           void* d_temp, size_t* temp_bytes, void* stream);

/* Windowed banded Gotoh score (SURVEY 8a row b7, second half): rows [window_begin, min(window_end, pattern length)) of every
 * alignment still alive, the (H, F) band carried between calls in d_checkpoints (band_len short2 per alignment, clamped at
 * SHRT_MIN+32 when stored), the BestSink in d_score / d_sink (in/out) and the reference's bool result in d_alive
 * (0 = text shorter than pattern, or the band maximum can no longer reach d_min_score[i] + remaining_rows * match; such
 * alignments are skipped by later passes).  window_begin == 0 initialises score / sink / alive.  d_min_score may be NULL
 * (= INT_MIN: never give up).  Scoring a pattern in consecutive windows yields exactly nvb_banded_gotoh_score's result as long as
 * every H and F stored in a checkpoint lies in [SHRT_MIN+32, 32767]; a larger value wraps when stored, as in the reference (whose
 * checkpoints are short2 as well), and the later windows then follow the reference rather than the one-pass score.
 * Replaces aln::banded_alignment_score<BAND_LEN>(aligner, pattern, quals, text, min_score, window_begin, window_end, sink,
 * checkpoint) (nvbio/alignment/banded_inl.h:178-218, gotoh_banded_inl.h:132-199,616-634,706-739), the per-pass body of
 * BatchedBandedAlignmentScore<..., DeviceStagedThreadScheduler> (batched_banded_inl.h:170-241).  bands 3, 5, 7, 15, 31. */
int nvb_banded_gotoh_score_window(int band_len, int type, const nvb_gotoh_scheme* scheme,
                                  const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                                  uint32_t window_begin, uint32_t window_end, const int32_t* d_min_score,
                                  int16_t* d_checkpoints, int32_t* d_score, nvb_uint2* d_sink, uint8_t* d_alive, void* stream);

/* Banded Gotoh score with aln::Best2Sink<int32>(distinct_dist) (nvbio/alignment/sink.h:114-147, sink_inl.h:70-116) instead of BestSink: the
 * best alignment (last maximal report wins) and the best one whose text end is more than distinct_dist away from it -- the second-best
 * score a MAPQ estimate needs.  d_out6[6*i ..] = (score1, sink1.x, sink1.y, score2, sink2.x, sink2.y); unset entries keep the sink's
 * defaults (NVB_SINK_MIN, 0xFFFFFFFF).  Every report the reference makes reaches the sink in its order (LOCAL: every cell, row by row).
 * One alignment per thread on the int32 kernel; bands 3, 5, 7, 15, 31, 63. */
int nvb_banded_gotoh_score_best2(int band_len, int type, const nvb_gotoh_scheme* scheme,
                                 const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                                 uint32_t distinct_dist, int32_t* d_out6, void* stream);

/* Full-matrix (un-banded) Gotoh score (SURVEY 8f-3): every pattern against the WHOLE of its text.
 * d_score / d_sink = BestSink<int32>{score, (text end, pattern end)}; pattern and text lengths must be >= 1 and
 * `patterns->length` / `texts->length` must bound them (<= 65535; the text bound sizes the boundary-column scratch).
 * Replaces aln::alignment_score / aln::BatchedAlignmentScore<stream,DeviceThreadScheduler> with
 * GotohAligner<TYPE,SimpleGotohScheme> (default PatternBlockingTag; nvbio/alignment/alignment_inl.h:95-125,
 * gotoh/gotoh_inl.h:459-960, batched_inl.h:236-605) -- the DP sw-benchmark times (sw-benchmark.cu:592-641) and nvBowtie's
 * opposite-mate scoring.  LOCAL ties resolve in the reference's (8-column stripe, row, column) order.
 * d_quals (one byte per pattern symbol, indexed like the pattern offsets; may be NULL) and scheme->d_qual_table select the
 * quality-dependent substitution scores as in nvb_banded_gotoh_score; such batches run on the int32 kernel. */
int nvb_gotoh_score(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                    int32_t* d_score, nvb_uint2* d_sink, void* d_temp, size_t* temp_bytes, void* stream);

/* Same, with the number of alignments read from device memory (*d_n, clamped to n_max): lets a producer kernel decide
 * the batch size without a host round trip (the opposite-mate stage of nvb_seed_extend_paired). */
int nvb_gotoh_score_indirect(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts,
                             const uint32_t* d_n, uint32_t n_max,
                             int32_t* d_score, nvb_uint2* d_sink, void* d_temp, size_t* temp_bytes, void* stream);

/* Full-matrix Gotoh traceback: score + sink as nvb_gotoh_score, plus the alignment itself.
 *   d_ops[i*max_ops ..]  the backtracer's pushes in END -> START order (0 = SUBSTITUTION 'M', 1 = INSERTION 'I' (pattern symbol
 *                        against a gap), 2 = DELETION 'D'), d_n_ops[i] their number (may exceed max_ops: then truncated)
 *   d_source[i]          = (text begin, pattern begin) of the alignment; the soft clips of the pattern are
 *                          pattern_len - sink.y at the end and source.y at the start
 * Replaces aln::alignment_traceback<MAX_PATTERN_LEN,MAX_TEXT_LEN,CHECKPOINTS> with a Gotoh aligner (generic driver
 * nvbio/alignment/alignment_inl.h:365-530; state machine gotoh/gotoh_inl.h:1806-1871) and its batched form
 * BatchedAlignmentTraceback (batched_inl.h:607-860).  No checkpoints: d_temp holds the whole direction matrix, 4 bits per cell
 * (max_text_len * ceil(max_pattern_len/32) * 16 bytes per alignment). */
int nvb_gotoh_traceback(int type, const nvb_gotoh_scheme* scheme, const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                        int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                        uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops,
                        void* d_temp, size_t* temp_bytes, void* stream);

/* Banded Gotoh traceback (SURVEY 8f-4).  For i < n: score, sink (end cells) as nvb_banded_gotoh_score, plus the
 * source (start cells) and the alignment as the backtracer's pushes in END -> START order, one byte per op
 * (0 = SUBSTITUTION 'M', 1 = INSERTION 'I', 2 = DELETION 'D'; nvbio::aln::DirectionVector) at d_ops[i*max_ops ..];
 * d_n_ops[i] = number of ops (ops beyond max_ops are counted, not stored).  An alignment takes one op per pattern row (M or I)
 * plus one per D, and its M and D ops consume at most pattern length + band_len - 1 text columns, so max_ops >= 2 * pattern length
 * + band_len always suffices; pattern length + band_len does not when an alignment pairs insertions with deletions.  The soft clips the reference passes to Backtracer::clip are (pattern_len - sink.y) and source.y.
 * `patterns->length` must bound the pattern lengths (it sizes the per-alignment direction matrix in d_temp).
 * Replaces aln::banded_alignment_traceback<BAND_LEN,MAX_PATTERN_LEN,CHECKPOINTS> and
 * BatchedBandedAlignmentTraceback (nvbio/alignment/banded_inl.h:352-489, gotoh/gotoh_banded_inl.h:763-962,
 * batched_banded_inl.h:248-451): instead of 32-row checkpoints + window recomputation the whole 4-bit direction
 * matrix of every alignment is kept in HBM and walked once. */
int nvb_banded_gotoh_traceback(int band_len, int type, const nvb_gotoh_scheme* scheme,
                               const nvb_string_set* patterns, const uint8_t* d_quals, const nvb_string_set* texts, uint32_t n,
                               int32_t* d_score, nvb_uint2* d_sink, nvb_uint2* d_source,
                               uint8_t* d_ops, uint32_t max_ops, uint32_t* d_n_ops,
                               void* d_temp, size_t* temp_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Index construction on the device (SURVEY 8f-1; needed to run any of the above on synthetic data)
 * ------------------------------------------------------------------------------------------- */

/* Build occ + interleave: d_bwt holds n 2-bit big-endian BWT symbols (ceil(n/64)*4 words, padding
 * ignored); writes ceil(n/64) 32-byte blocks to d_bwt_occ and the L2 table to h_L2 (synchronises).
 * Replaces nvbio::build_occurrence_table<2,64> + the interleave loop
 * (nvbio/fmindex/rank_dictionary_inl.h:42-77, nvbio/io/fmindex/fmindex_impl.cu:263-331).
 * NVB_E_INVALID for n > NVB_FM_MAX_LENGTH. */
int nvb_fm_build_occ(const uint32_t* d_bwt, uint32_t n, void* d_bwt_occ, uint32_t h_L2[5],
                     void* d_temp, size_t* temp_bytes, void* stream);

/* Suffix-sort a 2-bit big-endian packed text of n symbols on the device and emit the BWT (nvbio
 * convention: `$` row removed, nvbio/fmindex/bwt.h:51-63), the primary row, the sampled SA
 * (every sa_interval-th row, ssa[0]=0xFFFFFFFF; sa_interval 0 means 16) and optionally the full SA with
 * the `$` row (n+1 entries, d_sa may be NULL).
 * d_bwt must hold ceil(n/64)*4 words, d_ssa (n+I)/I words.  Synchronises.  NVB_E_INVALID for n > NVB_FM_MAX_LENGTH. */
int nvb_fm_build_bwt(const uint32_t* d_text, uint32_t n, uint32_t* d_bwt, uint32_t* h_primary,
                     uint32_t* d_ssa, uint32_t sa_interval, uint32_t* d_sa,
                     void* d_temp, size_t* temp_bytes, void* stream);

/* Fill d_ktab[4^k] with match() of every k-mer (level by level: 4^k * 4/3 LF steps in total).
 * k in [1,16] (8.6 GB at k=15, 34 GB at k=16).  fmi->d_ktab / ktab_k are ignored on input. */
int nvb_fm_build_ktab(const nvb_fm_index* fmi, uint32_t k, nvb_uint2* d_ktab, void* stream);

/* The same table with 16-byte entries {x, y, SA[x], SA[y]} (d_ktab16: 4^k * 16 bytes, 16-byte aligned; 69 GB at k = 16 -- HBM capacity
 * traded for dependent gathers).  The SA values are filled for ranges of one row (x == y) or two (y == x + 1) and need the full suffix array
 * (fmi->sa_interval == 1), else NVB_E_UNSUPPORTED.  Use with nvb_fm_index.d_ktab = d_ktab16, ktab_located = 1. */
int nvb_fm_build_ktab_located(const nvb_fm_index* fmi, uint32_t k, void* d_ktab16, void* stream);

/* nvb_fm_build_ktab_located + text context: for every one-row entry the unused last word is filled with the (up to) 16 symbols of
 * d_text (2-bit big-endian, the text the index was built from) that precede SA[x], symbol SA[x]-1 in the two lowest bits; two-row
 * entries are packed as described at nvb_fm_index.ktab_located.  Use with nvb_fm_index.d_ktab = d_ktab16, ktab_located = 2. */
int nvb_fm_build_ktab_context(const nvb_fm_index* fmi, uint32_t k, const uint32_t* d_text, void* d_ktab16, void* stream);

/* The context table with 32-byte entries, one DRAM sector each (d_ktab32: 4^k * 32 bytes, 32-byte aligned; 34.4 GB at k = 15).  Words
 * 0-3 of an entry are what nvb_fm_build_ktab_context writes, except for k-mers with 3 to 8 occurrences (rows x..y), which use the
 * words that format leaves zero.  With ctxN(r) = the (up to) N symbols of d_text before SA[r], symbol SA[r]-1 in the two lowest bits:
 *     3 rows:    {x, y, SA[x], SA[x+1], SA[x+2], ctx16(x), ctx16(x+1), ctx16(x+2)}
 *     4 rows:    {x, y, ctx8(x) | ctx8(x+1) << 16, ctx8(x+2) | ctx8(x+3) << 16, SA[x], SA[x+1], SA[x+2], SA[x+3]}
 *     5-8 rows:  {x, y, ctx8 of the rows two per word (row x in the low half of word 2, x+1 in its high half, ...), 0, ...}
 * Other entries have zero in words 4-7.  Needs the full suffix array (fmi->sa_interval == 1, fmi->d_ssa), else NVB_E_UNSUPPORTED;
 * fmi->d_ktab / ktab_k / ktab_located are ignored.  Uses no memory beyond the table.  Use with nvb_fm_index.d_ktab = d_ktab32,
 * ktab_located = 4 (5 with d_rows). */
int nvb_fm_build_ktab_wide(const nvb_fm_index* fmi, uint32_t k, const uint32_t* d_text, void* d_ktab32, void* stream);

/* Per-row array of an index with the full suffix array: d_rows[r] = {SA[r], the (up to) 16 symbols of d_text before SA[r], symbol SA[r]-1
 * in the two lowest bits} for r in [0, length] ((length + 1) * 8 bytes: 15.2 GB at 1.9 Gbp).  Row 0 (SA = 0xFFFFFFFF) gets context 0,
 * a row with SA[r] < 16 the SA[r] symbols there are.  Needs fmi->sa_interval == 1 and fmi->d_ssa, else NVB_E_UNSUPPORTED; fmi's table
 * fields are ignored.  Use with a context table (nvb_fm_build_ktab_context) as nvb_fm_index.d_rows = d_rows, ktab_located = 3. */
int nvb_fm_build_rows(const nvb_fm_index* fmi, const uint32_t* d_text, nvb_uint2* d_rows, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Seed + extend composition (the fmmap / nvBowtie hot loop: seeds -> match -> locate -> window ->
 * banded Gotoh -> best score per read; nvbio examples/fmmap/fmmap.cu:255-400)
 * ------------------------------------------------------------------------------------------- */
typedef struct nvb_seed_extend_params {
    uint32_t seed_len;        /* 20 (nvBowtie local) / 22 (fmmap)                                    */
    uint32_t seed_interval;   /* 10 for 150 bp: int(1 + 0.75*sqrtf(150)) evaluated on the host        */
    uint32_t band_len;        /* 31 */
    uint32_t type;            /* NVB_LOCAL */
    uint32_t both_strands;    /* 1: also seed/extend the reverse complement of every read           */
    uint32_t max_seed_hits;   /* ranges wider than this contribute only their first max_seed_hits rows */
    uint32_t dedup_jobs;      /* 1: hits of a read that define the same (strand, window) alignment are scored once and
                                 the result copied to each of them (bit-identical per-hit outputs, fewer cells)       */
    nvb_gotoh_scheme scheme;
    const uint8_t* d_read_quals; /* optional base qualities, one byte per read symbol: the quality of symbol p of read r is
                                    d_read_quals[offset of read r in symbols + p] (the indexing of nvb_banded_gotoh_score's
                                    d_quals); used with scheme.d_qual_table (nvBowtie's scoring); NULL = none        */
} nvb_seed_extend_params;

/* reads: n_reads strings (2- or 4-bit).  genome: 2-bit big-endian packed text of fmi->length symbols.
 * Outputs: d_best_score[n_reads] (INT_MIN when a read has no hit), d_best_pos[n_reads] = genome
 * coordinate of the best alignment's end (window begin + sink.x; 0xFFFFFFFF when none).
 * A job the banded DP reports empty (sink.x == 0xFFFFFFFF, score NVB_SINK_MIN: its window is shorter than the read, as for a read
 * running more than band_len/2 symbols past the genome's end) is not an alignment: it keeps its per-hit outputs and counts as a hit,
 * but is never a read's best or second-best alignment nor a paired-end candidate.  A read whose jobs are all empty is unaligned
 * (INT_MIN, 0xFFFFFFFF; n_ops 0 and MAPQ 0 in the calls below; an unaligned mate in the paired ones).
 * Optional per-hit outputs (may be NULL) of capacity hit_capacity: d_hit_read (string id = read*strands
 * + strand), d_hit_window (begin,end), d_hit_score, d_hit_sink; d_n_hits[0] receives the number of hits
 * kept (<= hit_capacity), d_n_hits[1] the number found and d_n_hits[2] the number of distinct alignment jobs
 * actually scored (device counters, no host round trip).
 * Returns NVB_E_TEMP_SIZE with the needed size when d_temp is NULL/too small. */
int nvb_seed_extend(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    void* d_temp, size_t* temp_bytes, void* stream);

/* Optional alignment of every read's best hit (what nvBowtie's banded_traceback_best produces for SAM output,
 * aligner_best_approx.h:300-500): the banded traceback of the best (strand, window) job of each read.
 *   d_ops[r*max_ops ..]  ops in END -> START order (0 M, 1 I, 2 D), d_n_ops[r] their number (0 when the read has no hit)
 *   d_begin[r]           = (genome coordinate of the alignment's first text symbol, first aligned read symbol)
 *   d_strand[r]          = 0 forward, 1 reverse complement (the read symbols are those of that strand's string)
 * Call with the same arguments as nvb_seed_extend plus this struct; temp size grows by the direction matrices. */
typedef struct nvb_best_alignment_out {
    uint8_t*   d_ops;
    uint32_t   max_ops;
    uint32_t*  d_n_ops;
    nvb_uint2* d_begin;
    uint8_t*   d_strand;
} nvb_best_alignment_out;

int nvb_seed_extend_traceback(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    void* d_temp, size_t* temp_bytes, void* stream);

/* Second-best distinct alignment and mapping quality of every read (single end; what nvBowtie's score_reduce_kernel and BowtieMapq2
 * produce, nvBowtie/bowtie2/cuda/reduce_inl.h:73-152, mapq.h:142-331).  The candidates of read r are the alignments the call scores:
 * its distinct (strand, window) jobs, or every kept hit when per-hit outputs are requested; each has a score s, a strand t, an end p
 * (window begin + sink.x, like d_best_pos) and a tie index (its first hit).  A candidate is distinct from the best alignment (strand bt,
 * end bp) when t != bt or p lies outside [bp - min(bp, len/2), bp + len/2] (len = the read's length; io::distinct_alignments).
 * The second best is the distinct candidate with s >= d_min_score[len] and the largest s, ties to the smallest tie index -- one answer
 * whatever the job order, path or de-duplication (nvBowtie's order-dependent hit-by-hit reduction can differ, see DESIGN.md).
 *   d_second_score[r]   INT_MIN when there is none;  d_second_pos[r]  its end, 0xFFFFFFFF when none;  d_second_strand[r]  0 when none
 *   d_mapq[r]           BowtieMapq2 of an unpaired read with perfect_score(len) = len * match_bonus, min_score(len) = d_min_score[len]
 *                       and the end-to-end (monotone) branch when match_bonus == 0; 0 for reads without an alignment
 * d_min_score is the caller's --score-min evaluated on the host for every length 0 .. max_read_len (nvbio_b200.MapqParams does it
 * for nvBowtie's SimpleFunc).  Call with the same arguments as nvb_seed_extend_traceback; best_alignment may be NULL.  The best
 * alignment outputs are those of nvb_seed_extend.  Returns NVB_E_INVALID when mapq, mapq_out, d_min_score, d_second_score or d_mapq
 * is NULL, or max_read_len < reads->length; the temp size grows by 8 bytes per read. */
typedef struct nvb_mapq_params {
    const int32_t* d_min_score;   /* device, [max_read_len + 1]: minimum valid score of a read of each length (host-evaluated --score-min) */
    uint32_t       max_read_len;
    int32_t        match_bonus;   /* perfect_score(len) = len * match_bonus; 0 = end-to-end scheme (BowtieMapq2's monotone branch) */
} nvb_mapq_params;
typedef struct nvb_mapq_out {
    int32_t*  d_second_score;     /* [n_reads], required */
    uint32_t* d_second_pos;       /* [n_reads], may be NULL */
    uint8_t*  d_second_strand;    /* [n_reads], may be NULL */
    uint8_t*  d_mapq;             /* [n_reads], required */
} nvb_mapq_out;

int nvb_seed_extend_mapq(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    const nvb_mapq_params* mapq, const nvb_mapq_out* mapq_out,
                    void* d_temp, size_t* temp_bytes, void* stream);

/* Reseeding rounds (single end; nvBowtie's -R / --rep-seeds, params.cpp:126-127, aligner_best_approx.h:206-283; DESIGN.md 3.18).
 * Call with the arguments of nvb_seed_extend_mapq (best_alignment, mapq and mapq_out each optional; mapq and mapq_out together) plus:
 *   Round 0 is every read with exactly nvb_seed_extend's seeds; round r >= 1 covers only the reads flagged after round r - 1, in read
 *   order.  Each string (forward, and the reverse complement with both_strands) is seeded at o_r + k*I for every k with o_r + k*I + L <= its
 *   length, o_r = r * floor(I / (max_reseed + 1)), I = seed_interval, L = seed_len.  A read's base qualities go with it into every round.
 *   Flag rule after round r < max_reseed, over the round's seeds of both strings: range_count = the seeds with a non-empty SA range (a seed
 *   with an N has an empty one), range_sum = the sum of their full range sizes y - x + 1 (not capped by max_seed_hits), both in wrapping
 *   uint32 arithmetic as nvb_map_seeds'.  A read is flagged when range_count == 0, range_sum >= rep_seeds * range_count, or its best
 *   alignment over rounds 0 .. r is below d_min_score[len] or absent.
 *   A read's candidates are the union of its rounds' jobs.  The best alignment: higher score, then earlier round, then nvb_seed_extend's tie
 *   index within the round (a later round replaces the best only with a strictly higher score).  Second best, MAPQ, distinctness and the
 *   traceback follow nvb_seed_extend_mapq's rules over that union with the tie index ordered by (round, tie); the results do not depend on
 *   the path, the de-duplication, the exact shortcut or the seed split.  A job found in several rounds may be scored in each.
 *   Per-hit outputs: round-major, within a round nvb_seed_extend's order for the round's reads; d_hit_read is the original string id
 *   (read * strands + strand).  hit_capacity is shared by all rounds (round r keeps at most hit_capacity minus the hits kept before it).
 *   d_n_hits = (hits kept, hits found, distinct jobs), each summed over the rounds.
 *   Host round trip: after every round but the last the number of flagged reads is read back (one stream synchronisation per round, so the
 *   call returns after rounds 0 .. max_reseed - 1 have run), to size the next round's grids and to stop when no read is flagged.
 *   The temp size covers every read flagged in every round.
 * NVB_E_INVALID before any CUDA call: reseed == NULL, d_min_score == NULL, max_read_len < reads->length, max_reseed > 254, or max_reseed > 0
 * with seed_interval < max_reseed + 1 -- a deliberate deviation from nvBowtie, whose shifted seeds would all repeat round 0's there; the
 * other checks are nvb_seed_extend_mapq's.  With max_reseed == 0 every output is that of nvb_seed_extend[_traceback|_mapq]. */
typedef struct nvb_reseed_params {
    uint32_t       max_reseed;    /* nvBowtie -R: rounds after the first; 0 = exactly nvb_seed_extend[_traceback|_mapq]   */
    uint32_t       rep_seeds;     /* nvBowtie --rep-seeds (300)                                                          */
    const int32_t* d_min_score;   /* device [max_read_len + 1]: a read is aligned when its best score >= d_min_score[len] */
    uint32_t       max_read_len;
} nvb_reseed_params;
typedef struct nvb_reseed_out {
    uint8_t*  d_rounds;           /* [n_reads] or NULL: the number of rounds read r was seeded in, 1 .. max_reseed + 1    */
    uint32_t* d_active;           /* [max_reseed + 1] or NULL: the number of reads seeded in each round                   */
} nvb_reseed_out;

int nvb_seed_extend_reseed(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    const nvb_mapq_params* mapq, const nvb_mapq_out* mapq_out,
                    const nvb_reseed_params* reseed, const nvb_reseed_out* reseed_out,
                    void* d_temp, size_t* temp_bytes, void* stream);

/* Up to k distinct alignments of every read, each traced (single end; nvBowtie's all-mapping mode, --all / -a, params.cpp:140-142,
 * aligner_all.h:49-235 and 278-690, with the per-read limit of Bowtie2's -k).  Call with the arguments of nvb_seed_extend_mapq, with
 * best_alignment == NULL; the best, second-best and MAPQ outputs are exactly those of nvb_seed_extend_mapq for the same inputs.
 *   Candidates of read r: the alignments nvb_seed_extend_mapq's second-best rule sees (score s, strand t, end p = window begin + sink.x, tie
 *   index), without the empty jobs and without those with s < d_min_score[len] -- every alignment the reference's all mode reports reaches
 *   that score (score_all_inl.h:141-150).
 *   Selection: the candidates in descending (s, -tie) order (make_best_key); a candidate (p, t) is admitted when it is distinct from every
 *   alignment (a.end, a.strand) admitted before it -- distinct_alignment(p, t, a.end, a.strand, len), t != a.strand or p outside
 *   [a.end - min(a.end, len/2), a.end + len/2] (io::distinct_alignments, nvbio/io/alignments_inl.h:33-47); the walk stops after
 *   max_per_read admissions (0: none).  So rank 0 is nvb_seed_extend's best alignment when that reaches the min score (a read whose best
 *   is below it has no alignment here), and for max_per_read != 1 rank 1 is nvb_seed_extend_mapq's second-best alignment.
 *   Output: read order, and rank order within a read.  d_first is the exclusive scan of the per-read counts, written whole; read r's
 *   alignments [d_first[r], d_first[r + 1]) are stored only if d_first[r + 1] <= capacity, so the stored reads are a prefix.  d_count =
 *   (alignments stored, wanted), as d_n_rescue.  Alignment i: d_read[i], d_score[i], d_pos[i] (its end), and in `alignment` its banded
 *   traceback as nvb_seed_extend_traceback writes a read's (ops END -> START at d_ops[i * max_ops ..], d_n_ops[i], d_begin[i] = (genome
 *   coordinate of the first aligned text symbol, first aligned read symbol), d_strand[i]): equal to nvb_banded_gotoh_traceback of its
 *   (strand, window) job alone.  Entries at or beyond d_count[0] are not written.  No host round trip.
 *   Deliberate deviations from nvBowtie (DESIGN.md section 3.16): it de-duplicates only identical (read, strand, seed diagonal) hits
 *   (aligner_all.h:496-553), so one locus reached on two diagonals is reported twice -- here the distinct rule suppresses that; and the
 *   per-read limit max_per_read.
 * NVB_E_INVALID (before any CUDA call) for a NULL mapq, all_params or all_out, a NULL d_first / d_read / d_score / d_pos / d_count or
 * alignment.d_ops / d_n_ops / d_begin / d_strand, best_alignment != NULL, alignment.max_ops == 0, or the checks of nvb_seed_extend_mapq;
 * NVB_E_UNSUPPORTED for reads->length > 512 (as the paired traceback).  The alignments are traced in ceil(capacity / n_reads) slices of
 * at most n_reads (each a few kernel launches; one past the stored alignments does no work), so the
 * temp size grows by the traceback's share of nvb_seed_extend_traceback plus about 24 bytes per unit of hit_capacity, 16 bytes per
 * alignment slot and 12 bytes per read. */
typedef struct nvb_all_params {
    uint32_t max_per_read;             /* k; 0 = every distinct alignment (nvBowtie --all) */
    uint32_t capacity;                 /* alignment slots of the per-alignment outputs */
} nvb_all_params;
typedef struct nvb_all_out {
    uint32_t* d_first;                 /* [n_reads + 1] read r's alignments are [d_first[r], d_first[r + 1]); always written whole */
    uint32_t* d_read;                  /* [capacity] the read of alignment i */
    int32_t*  d_score;                 /* [capacity] */
    uint32_t* d_pos;                   /* [capacity] end = window begin + sink.x, as d_best_pos */
    nvb_best_alignment_out alignment;  /* [capacity] ops / n_ops / begin / strand, as nvb_seed_extend_traceback */
    uint32_t* d_count;                 /* [2] alignments stored, wanted */
} nvb_all_out;

int nvb_seed_extend_all(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_reads,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    int32_t* d_best_score, uint32_t* d_best_pos,
                    uint32_t* d_n_hits, uint32_t* d_hit_read, nvb_uint2* d_hit_window,
                    int32_t* d_hit_score, nvb_uint2* d_hit_sink,
                    const nvb_best_alignment_out* best_alignment,
                    const nvb_mapq_params* mapq, const nvb_mapq_out* mapq_out,
                    const nvb_all_params* all_params, const nvb_all_out* all_out,
                    void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * Paired-end composition (BASELINE configs[4] shape; nvBowtie best_approx paired: anchor scoring + opposite-mate full DP,
 * nvBowtie/bowtie2/cuda/aligner_best_approx_paired.h, score_opposite_inl.h:90-266, alignment_utils.h:62-95 PE_POLICY_FR).
 *
 * reads = 2*n_pairs strings: mate 1 of pair p at index p, mate 2 at index n_pairs + p.  Every mate is seeded and extended
 * on its own (nvb_seed_extend with both_strands = 1, which is required).  Per pair, under the default FR policy (the other policies,
 * --no-overlap, discordant pairs and --no-mixed: policy / flags below):
 *   - if both mates have a best alignment, on opposite strands, the forward one starting at or before the reverse one,
 *     ending at or before it, and the fragment [begin of the forward mate, end of the reverse mate) has a length in
 *     [min_frag, max_frag]: the pair is CONCORDANT as it stands (alignment begin := end - read length, clamped at 0);
 *   - otherwise every mate that has an alignment (score >= min_mate_score) acts as anchor and the OTHER mate is searched
 *     with the full-matrix Gotoh DP (nvb_gotoh_score, same type and scheme) where the FR policy puts it: anchor forward at
 *     [b, e) -> the reverse complement of the other mate in [b, min(b + max_frag, genome length)); anchor reverse ->
 *     the other mate forward in [max(e - max_frag, 0), e)  (score_opposite_inl.h:177-191 with pe_overlap).  A rescue whose
 *     score reaches min_mate_score yields a candidate pair; the candidate with the larger score sum wins (tie: mate 1 as
 *     anchor).  No candidate: the pair is UNPAIRED and each mate keeps its own best alignment.
 * A mate's alignment BEGIN is taken as (end - read length, clamped at 0), not from a traceback: with soft clips or indels the true
 * start differs by a few bases, so pairs within that distance of min_frag / max_frag may be classified differently from a
 * caller that traces every alignment (nvBowtie does); callers that need the exact extent of both mates, rescued ones included, can
 * call nvb_seed_extend_paired_traceback and re-check those pairs.
 * At most rescue_capacity full-DP jobs are run per call (in pair order; d_n_rescue[1] reports how many were wanted).
 * Outputs (mate m of pair p at index m*n_pairs + p): d_pair_score (sum of the two mates' scores, INT_MIN when unpaired),
 * d_pair_flags (NVB_PAIR_*), d_mate_score (INT_MIN = unaligned), d_mate_pos (genome coordinate one past the last aligned
 * base, 0xFFFFFFFF = unaligned), d_mate_strand (0 forward, 1 reverse complement). */
/* Orientation and options (policy / flags; nvBowtie's --fr / --rf / --ff / --rr, --no-overlap, --no-mixed, --no-discordant,
 * params.cpp:160-170).  Zero-initialise the struct (memset or `= {0}`): every field added later means "as before" at zero, and the
 * zeroed policy and flags are the FR pairing above, bit for bit.
 *   policy: NVB_PE_FR (0), NVB_PE_RF, NVB_PE_FF or NVB_PE_RR.  The framing of anchor mate a aligned on strand t is nvBowtie's
 *     frame_opposite_mate(policy, a, anchor_fw = (t == 0)) (alignment_utils.h:61-98): whether the other mate lies to the left or the
 *     right of the anchor, and its strand.  (nvBowtie numbers io::PE_POLICY_* FF 0, FR 1, RF 2, RR 3; here 0 is FR so that a zeroed
 *     struct keeps today's pairing.)  Concordance, with (left, o) the framing of mate 1: mate 2 is on strand o and, with L / R the left
 *     / right mate as framed, L.b <= R.b, L.e <= R.e, R.e > L.b and min_frag <= R.e - L.b <= max_frag -- the FR test above for NVB_PE_FR.
 *     The rescue aligns the other mate's strand-o string against [b, min(b + max_frag, genome length)) when it lies to the right of an
 *     anchor at [b, e), against [max(e - max_frag, 0), e) when it lies to the left; the rescued mate gets strand o.
 *   NVB_PE_NO_OVERLAP: concordance also needs L.e <= R.b, and the rescue window starts at e (right) / ends at b (left).
 *   NVB_PE_DISCORDANT (requires mapq / mapq_out): after the rescue, an UNPAIRED pair whose two mates both have a best alignment with
 *     score >= d_min_score[len] and no single-end second alignment (second score INT_MIN: both unique) becomes NVB_PAIR_DISCORDANT
 *     (nvBowtie's mark_discordant, aligner_init.cu:459-482).  Off at zero, although nvBowtie's default is on: a zeroed struct keeps
 *     today's outputs.  A discordant pair reports pair score s1 + s2, the mates' single-end alignments and tracebacks, no second pair,
 *     and both mates' MAPQ = BowtieMapq2(s1 + s2, no second, perfect (len1 + len2) * match_bonus, min d_min_score[len1] +
 *     d_min_score[len2]), as MapqFunctorPE scores it.
 *   NVB_PE_NO_MIXED: after the discordant marking, both mates of every pair still UNPAIRED are reported unaligned in every output
 *     (score INT_MIN, pos 0xFFFFFFFF, strand 0, MAPQ 0, mate second score INT_MIN, n_ops 0, begin (0xFFFFFFFF, 0xFFFFFFFF)).  With
 *     NVB_PE_DISCORDANT also set, discordant pairs are still reported (Bowtie2's meaning of the two options).  Deliberate deviation:
 *     nvBowtie tracks no unpaired alignment under --no-mixed and so never marks a discordant pair there.
 * NVB_E_INVALID (before any CUDA call) for policy > 3 or an unknown flag bit, and for NVB_PE_DISCORDANT without mapq / mapq_out. */
typedef struct nvb_pair_params {
    uint32_t min_frag, max_frag;
    int32_t  min_mate_score;
    uint32_t rescue_capacity;
    uint32_t policy;            /* NVB_PE_FR (0), NVB_PE_RF, NVB_PE_FF, NVB_PE_RR */
    uint32_t flags;             /* NVB_PE_NO_OVERLAP | NVB_PE_DISCORDANT | NVB_PE_NO_MIXED */
} nvb_pair_params;
#define NVB_PE_FR               0u
#define NVB_PE_RF               1u
#define NVB_PE_FF               2u
#define NVB_PE_RR               3u
#define NVB_PE_NO_OVERLAP       1u
#define NVB_PE_DISCORDANT       2u
#define NVB_PE_NO_MIXED         4u
typedef struct nvb_pair_out {
    int32_t*  d_pair_score;     /* [n_pairs]   */
    uint32_t* d_pair_flags;     /* [n_pairs]   */
    int32_t*  d_mate_score;     /* [2*n_pairs] */
    uint32_t* d_mate_pos;       /* [2*n_pairs] */
    uint8_t*  d_mate_strand;    /* [2*n_pairs] */
    uint32_t* d_n_rescue;       /* [2] full-DP jobs run, wanted (may be NULL) */
} nvb_pair_out;
#define NVB_PAIR_UNPAIRED       0u
#define NVB_PAIR_CONCORDANT     1u    /* the mates' independent best alignments form a proper pair under the policy */
#define NVB_PAIR_RESCUED_MATE1  2u    /* mate 1 was placed by the opposite-mate DP next to mate 2's alignment */
#define NVB_PAIR_RESCUED_MATE2  4u
#define NVB_PAIR_DISCORDANT     8u    /* not concordant, both mates aligned uniquely (NVB_PE_DISCORDANT): a pair without the proper-pair bit */

int nvb_seed_extend_paired(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream);

/* Second-best pair and mapping quality of every mate (paired end; nvBowtie's BowtieMapq2 on BestPairedAlignments as MapqFunctorPE runs it,
 * aligner_best_approx_paired.h:50-96, mapq.h:155-170).  The pairing is that of nvb_seed_extend_paired, whose outputs this call returns
 * unchanged for the same inputs; call the pair it reports P*.
 *   Mate candidates: those of nvb_seed_extend_mapq for that read (score s, strand t, end e, tie index), begin b = e - len clamped at 0,
 *   and only those with s >= d_min_score[len].  Candidates with equal (strand, end) are merged into the one with the highest (s, -tie).
 *   Candidate pairs of a CONCORDANT or RESCUED pair: (1) every combination of one candidate of each mate that is concordant under the
 *   policy and flags (the concordance test of nvb_pair_params), score s1 + s2; (2) every opposite-mate job the call ran
 *   (j < rescue_capacity) whose score rs reaches min_mate_score and d_min_score[len]: the anchor's single-end best plus the rescued
 *   alignment (end = window begin + sink.x, strand as the policy frames it), score = anchor score + rs, the rescued mate's tie index
 *   0xFFFFFFFF.  Rescues exist only for pairs that were not concordant as they stood.  A DISCORDANT pair has no candidate pair.
 *   A candidate pair is not distinct from P* when both of its mates fail the single-end test against P*'s matching mate (same strand,
 *   end within len/2).  The second-best pair is the distinct candidate pair with the largest score, ties to the smaller mate-1 tie index,
 *   then the smaller mate-2 tie index -- one answer whatever the job order, path, de-duplication, exact shortcut or seed split.
 *   A distinct pair may score ABOVE P*: two non-best alignments can be concordant where the bests are not and the rescue missed them.
 *   It is still reported as the second pair (a low MAPQ); how the best pair is chosen does not change.
 *   d_mate_mapq of a CONCORDANT or RESCUED pair, both mates: BowtieMapq2 with best = pair score, the second pair's score when there is
 *   one, perfect = (len1 + len2) * match_bonus, min = d_min_score[len1] + d_min_score[len2], monotone when match_bonus == 0; of a
 *   DISCORDANT pair the same without a second.  Mates of an UNPAIRED pair: their single-end MAPQ (nvb_seed_extend_mapq on the 2n reads),
 *   0 under NVB_PE_NO_MIXED; an unaligned mate: 0.
 * Mate m of pair p at index m * n_pairs + p, as in nvb_pair_out.  Validation as nvb_seed_extend_paired and nvb_seed_extend_mapq:
 * NVB_E_INVALID when mapq, mapq_out, d_min_score, d_second_pair_score or d_mate_mapq is NULL, or max_read_len < reads->length.
 * The temp size grows by about 36 bytes per unit of hit_capacity plus 28 bytes per read; nvb_seed_extend_paired does not carve it. */
typedef struct nvb_pair_mapq_out {
    int32_t*  d_second_pair_score;   /* [n_pairs], required; INT_MIN when there is no second pair */
    uint32_t* d_second_mate_pos;     /* [2*n_pairs], may be NULL; each mate's end in the second pair, 0xFFFFFFFF when none */
    uint8_t*  d_second_mate_strand;  /* [2*n_pairs], may be NULL; 0 when none */
    int32_t*  d_mate_second_score;   /* [2*n_pairs], may be NULL; every mate's single-end second score (INT_MIN when none) */
    uint8_t*  d_mate_mapq;           /* [2*n_pairs], required */
} nvb_pair_mapq_out;

int nvb_seed_extend_paired_mapq(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    const nvb_mapq_params* mapq, const nvb_pair_mapq_out* mapq_out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream);

/* The alignment of both mates (what nvBowtie's paired aligner traces for SAM output, aligner_best_approx_paired.h:404-486).  Pairing,
 * pair outputs and, with mapq / mapq_out (both NULL or both set), the MAPQ outputs are exactly those of nvb_seed_extend_paired /
 * nvb_seed_extend_paired_mapq for the same inputs; concordance still uses begin = end - length.  mate_alignment is required and laid out
 * over the 2*n_pairs mates (mate m of pair p at index m * n_pairs + p), its fields meaning what they mean in nvb_best_alignment_out;
 * d_strand may be NULL (d_mate_strand holds the same).  Per mate:
 *   - unaligned (a mate of an UNPAIRED pair under NVB_PE_NO_MIXED included): n_ops = 0, begin = (0xFFFFFFFF, 0xFFFFFFFF);
 *   - keeping its own single-end best (CONCORDANT, DISCORDANT and UNPAIRED pairs, the anchor of a rescued pair): the banded traceback of that
 *     best (strand, window) job, equal to what nvb_seed_extend_traceback reports for the read when the 2*n_pairs mates run single end;
 *   - rescued (NVB_PAIR_RESCUED_MATE1 / 2): the full-matrix traceback of the winning opposite-mate job (the mate on the rescue strand
 *     against the rescue window), equal to nvb_gotoh_traceback of that job: begin = (window begin + source.x, source.y), the traced
 *     score and end are d_mate_score / d_mate_pos.
 * d_n_ops counts ops beyond max_ops without storing them.  NVB_E_INVALID when mate_alignment, d_ops, d_n_ops or d_begin is NULL,
 * max_ops is 0, only one of mapq / mapq_out is set, or a validation of the two calls above fails; NVB_E_UNSUPPORTED when
 * reads->length > 512 (nvBowtie's MAXIMUM_READ_LENGTH).  The temp size grows by the banded traceback's direction matrices for the
 * 2*n_pairs mates (reads->length * ceil(band_len / 8) * 4 bytes per mate) plus a slot pool of the rescue traceback: one slot of
 * (max_frag + 31) * 128 * ceil(ceil(reads->length / 32) / 8) bytes per resident warp (its occupancy times the SM count), whatever the
 * number of rescues. */
int nvb_seed_extend_paired_traceback(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    const nvb_best_alignment_out* mate_alignment,
                    const nvb_mapq_params* mapq, const nvb_pair_mapq_out* mapq_out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream);

/* Reseeding rounds before pairing (paired end; nvBowtie's -R / --rep-seeds, params.cpp:126-127, in its paired loop,
 * aligner_best_approx_paired.h:144-265; DESIGN.md 3.18).  Call with the arguments of nvb_seed_extend_paired_traceback, where
 * mate_alignment is optional here (NULL: no traceback) and mapq / mapq_out are optional together, plus reseed / reseed_out of
 * nvb_seed_extend_reseed:
 *   Rounds: the 2*n_pairs mates (mate m of pair p at index m*n_pairs + p) go through nvb_seed_extend_reseed's rounds as independent
 *   reads: round 0 seeds every mate; round r >= 1 seeds the mates flagged after round r - 1, in mate order, at reseed_offset(r, I,
 *   max_reseed) + k*I; base qualities go with each mate into every round; hit_capacity is shared by all rounds and d_n_hits gives the
 *   totals over all rounds, as there.
 *   Flag rule, seed statistics only: a mate goes on when range_count == 0 or range_sum >= rep_seeds * range_count over its round's seeds
 *   on both strings, in wrapping uint32 arithmetic (nvb_seed_extend_reseed's statistics).  Unlike the single-end call there is no
 *   "best alignment below its min score" term: nvBowtie's paired loop takes its reseed flags from map() alone (mapping_inl.h:586-588)
 *   and never marks unaligned mates (compare aligner_best_approx.h:267-271 with aligner_best_approx_paired.h:240-264); a mate whose
 *   partner aligns gets its second chance from the opposite-mate rescue.  reseed->d_min_score and max_read_len are not read (NULL / 0
 *   are accepted).
 *   Union, then pairing: every mate's best alignment is taken over the union of its rounds with the single-end rule (higher score, then
 *   earlier round, then tie index).  Pairing, concordance, the opposite-mate rescue, the paired MAPQ and the mate tracebacks then run
 *   once on that union, exactly as nvb_seed_extend_paired[_mapq|_traceback] run them on a single round: candidate tie indices order by
 *   (round, tie), so the second-best pair's tie-break is round-major; rescue_capacity and d_n_rescue keep their meaning (one rescue
 *   pass, in pair order).
 *   Deliberate deviation: nvBowtie scores the opposite mate for every anchor in every round; here the pairing decides once, after the
 *   last round -- the deviation nvb_seed_extend_paired already makes within a single round.  The policy and flags of pair_params apply
 *   to that one pairing; NVB_PE_DISCORDANT needs mapq / mapq_out.
 * Outputs: reseed_out->d_rounds is per mate, [2*n_pairs] in the mate layout above; d_active[r] counts the mates seeded in round r; every
 * other output means what it means in the three paired calls.  With max_reseed == 0 every output is that of nvb_seed_extend_paired,
 * _paired_mapq or _paired_traceback (whichever the optional groups select).  n_pairs == 0: NVB_OK with d_active zeroed.
 * Host round trip: one stream synchronisation per round after the first, as in nvb_seed_extend_reseed.
 * Validation before any CUDA call: NVB_E_INVALID as the paired calls (pair_params or out NULL, n_pairs > 0x3FFFFFFF, both_strands == 0,
 * max_frag == 0, min_frag > max_frag, a NULL required output field, only one of mapq / mapq_out set) and as nvb_seed_extend_reseed
 * (reseed == NULL, max_reseed > 254, max_reseed > 0 with seed_interval < max_reseed + 1); NVB_E_UNSUPPORTED when reads->length > 512
 * with mate_alignment. */
int nvb_seed_extend_paired_reseed(const nvb_fm_index* fmi, const uint32_t* d_genome,
                    const nvb_string_set* reads, uint32_t n_pairs,
                    const nvb_seed_extend_params* params, uint32_t hit_capacity,
                    const nvb_pair_params* pair_params, const nvb_pair_out* out,
                    const nvb_best_alignment_out* mate_alignment,
                    const nvb_mapq_params* mapq, const nvb_pair_mapq_out* mapq_out,
                    const nvb_reseed_params* reseed, const nvb_reseed_out* reseed_out,
                    uint32_t* d_n_hits, void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * Finishing traced alignments for SAM / BAM output (nvBowtie's finish_alignment_kernel, nvBowtie/bowtie2/cuda/traceback_inl.h:520-723,
 * and what its writers derive from the result, nvbio/io/output/output_sam.cpp:198-315, output_bam.cpp:66-91,
 * nvbio/io/output/output_utils.h:42-121).  One thread per alignment; no temp buffer; asynchronous on `stream`.
 *
 * Inputs: the outputs of nvb_seed_extend_traceback / nvb_seed_extend_paired_traceback as they are (`alignment`: d_ops, max_ops, d_n_ops,
 * d_begin, d_strand -- all required here; a paired caller passes d_mate_strand as d_strand) and the `reads` passed to that call: n
 * alignments, alignment i of read i (paired: n = 2 * n_pairs, mate m of pair p at m * n_pairs + p).  d_genome is the 2-bit big-endian
 * genome of genome_len symbols.  For strand 1 the read is reverse-complemented here (c < 4 ? 3 - c : c, as the traceback call does).
 * Per alignment, with len = the read's length and M, I, D = the numbers of columns of each op:
 *   - read span:    the aligned read symbols are [begin.y, begin.y + M + I) of the strand's string; the genome span is
 *                   [begin.x, begin.x + M + D);
 *   - CIGAR:        S(begin.y), the ops run-length encoded START -> END, S(len - begin.y - M - I); an S of length 0 is omitted.  BAM
 *                   encoding: run length << 4 | op (0 M, 1 I, 2 D, 4 S).  d_n_cigar counts the runs, also those beyond max_cigar, which
 *                   are not stored;
 *   - MD:Z:         as the SAM specification has it, [0-9]+(([A-Z]|\^[A-Z]+)[0-9]+)*: match counts, the REFERENCE base at a mismatch,
 *                   ^ and the reference bases of a deletion; a 0 separates adjacent tokens and stands at either end when needed;
 *                   insertions and soft clips do not appear.  Not NUL-terminated; d_md_len is the full length, also when it exceeds max_md
 *                   (then only max_md bytes are stored).  MD is at most 2 M + 3 D + 1 <= 3 n_ops + 1 bytes, so max_md = 3 max_ops + 1
 *                   and max_cigar = max_ops + 2 never truncate;
 *   - d_edits[4i..] = NM, XM, XO, XG: NM = mismatched M columns + I + D (clips excluded), XM = mismatched M columns, XO = number of I
 *                   runs + D runs, XG = the sum of (run length - 1) over those runs -- nvBowtie's edit distance (traceback_inl.h:579-660)
 *                   and analyze_md_string (output_utils.h:77-121);
 *   - a read N (4-bit reads) in an M column is a mismatch.  So is an M column at a genome coordinate >= genome_len: the banded DP reads
 *     past a window's end at the genome's end, and such an alignment still runs past the reference (the MD shows N there); clipping it
 *     is the caller's choice;
 *   - unaligned (n_ops == 0): n_cigar = 0, md_len = 0, edits all 0;
 *   - not finishable -- n_ops > max_ops (truncated by the traceback), begin.x == 0xFFFFFFFF with ops, an op byte > 2, or ops consuming more
 *     read symbols than len - begin.y: n_cigar = 0, md_len = 0, edits = (0xFFFFFFFF, 0, 0, 0).  Nothing is read or written out of bounds.
 * Deliberate deviations from nvBowtie (DESIGN.md): its MDS keeps the READ base of a mismatch (traceback_inl.h:644-645) and its SAM writer
 * prints that, omits the 0 between adjacent mismatches and before a leading one, appends a 0 after every deletion (output_sam.cpp:303)
 * and mis-merges match tokens longer than 255 (output_sam.cpp:263-265); here the MD is spec-conformant.  NM / XM / XO / XG equal nvBowtie's.
 * NVB_E_INVALID (before any CUDA call) for a NULL genome, reads, alignment, d_ops, d_n_ops, d_begin or d_strand, a NULL output array, or a
 * max_ops / max_cigar / max_md of 0; NVB_E_UNSUPPORTED for 8-bit reads. */
typedef struct nvb_finish_out {
    uint32_t* d_cigar;     /* [n * max_cigar]  BAM encoding (run length << 4 | op), op 0 M, 1 I, 2 D, 4 S; START -> END (genome order) */
    uint32_t  max_cigar;
    uint32_t* d_n_cigar;   /* [n]  runs, counted beyond max_cigar without storing them (as d_n_ops) */
    char*     d_md;        /* [n * max_md]  the MD:Z value, not NUL-terminated */
    uint32_t  max_md;
    uint32_t* d_md_len;    /* [n]  full length, also when > max_md (then only max_md bytes are stored) */
    uint32_t* d_edits;     /* [4 * n]  NM, XM, XO, XG */
} nvb_finish_out;

int nvb_finish_alignments(const uint32_t* d_genome, uint32_t genome_len,
                          const nvb_string_set* reads, uint32_t n,
                          const nvb_best_alignment_out* alignment,
                          const nvb_finish_out* out, void* stream);

/* -------------------------------------------------------------------------------------------
 * BAM alignment records of traced and finished alignments (the bam1_t wire layout of the SAM / BAM specification, what htslib's
 * bam_write1 writes after its BGZF framing, contrib/htslib/sam.c:335-361; nvBowtie's BAM and SAM writers, output_bam.cpp:234-446,
 * output_sam.cpp:354-530).  Asynchronous on `stream`, no host round trip; NVB_E_TEMP_SIZE protocol.
 *
 * Inputs (nvb_bam_in): the `reads` passed to the traceback call and optional base qualities d_read_quals (phred values indexed like the
 * read symbols); the traceback outputs d_n_ops / d_begin / d_strand; the nvb_finish_out of nvb_finish_alignments; the alignment score
 * (d_best_score, or d_mate_score when paired); optional d_mapq (or d_mate_mapq) and second score (d_second_score / d_mate_second_score);
 * paired only: d_pair_flags.  The contig table d_contig_begin[n_contigs + 1] holds concatenated coordinates, increasing, [0] = 0,
 * [n_contigs] = genome length.  Read names: bytes d_names, name j = [d_name_offsets[j], d_name_offsets[j + 1]), one per read when single
 * end and one per pair when paired, 1-254 printable bytes (longer names are cut at 254 bytes).
 * n alignments: single end, alignment i is read i and record i; paired (d_pair_flags != NULL, n even), alignment m * n / 2 + p (mate m of
 * pair p) becomes record 2p + m.
 *
 * Placement of an alignment, with M / D the columns of its CIGAR: span = [begin.x, begin.x + M + D); refID = upper_bound(contig_begin,
 * begin.x) - 1; pos = begin.x - contig_begin[refID].  It is MAPPED only if n_ops > 0, finish wrote it whole (NM != 0xFFFFFFFF, n_cigar <=
 * max_cigar and <= 65535, md_len <= max_md) and its span lies inside one contig (contig_begin[refID] <= begin.x < contig_begin[refID + 1]
 * and begin.x + M + D <= contig_begin[refID + 1]).  A span that crosses a contig boundary or runs past the genome (the genome-end M
 * columns of nvb_finish_alignments) is reported unmapped, as nvBowtie does (output_sam.cpp:457-464, output_bam.cpp:351-366); so the
 * mate sees an unmapped mate.
 * A mapped record:
 *   FLAG   0x10 on strand 1; paired: 0x1, 0x40 / 0x80 for mate 1 / 2, 0x2 when the pair is CONCORDANT or RESCUED and both mates are
 *          mapped (never for NVB_PAIR_DISCORDANT: such records carry 0x1, 0x40 / 0x80 and the mate fields without 0x2), 0x8 when
 *          the mate is unmapped, 0x20 when the mate is mapped on strand 1;
 *   MAPQ   d_mapq, 255 without it;   bin = reg2bin(pos, pos + M + D) (the specification's, hts_reg2bin(beg, end, 14, 5));
 *   CIGAR  the finish output;  SEQ the strand's string (strand 1 reverse-complemented, as the traceback saw it) in BAM's 4-bit
 *          =ACMGRSVTWYHKDBN code (A 1, C 2, G 4, T 8, N 15);  QUAL reversed for strand 1, all 0xFF without qualities;
 *   mate   mate mapped: next_refID / next_pos = its placement; TLEN = +-(max end - min begin) on the same contig (+ for the smaller
 *          begin, mate 1 on equal begins), 0 on different contigs.  Mate unmapped: its own placement, TLEN 0.  Single end: -1 / -1 / 0;
 *   tags   NM, AS, XS (only when the second score is given and not INT_MIN), XM, XO, XG, MD:Z (when not empty), in nvBowtie's order
 *          (output_sam.cpp:354-363); an integer tag has the type htslib's SAM parser picks: the smallest of c / s / i for a negative
 *          value, of C / S / I otherwise (contrib/htslib/sam.c:783-806), so a record is byte-identical to htslib's encoding of its SAM line.
 * An unmapped record: FLAG 0x4 plus the paired bits above (0x20 / 0x8 describe the mate), MAPQ 0, no CIGAR, no tags, SEQ / QUAL of the
 * read as given; with a mapped mate it takes the mate's refID / pos as its own and as next_refID / next_pos, bin = reg2bin(pos, pos + 1);
 * otherwise refID, pos, next_refID and next_pos are -1 and bin = 4680.
 * Deliberate deviations from nvBowtie's writers, which the specification decides (DESIGN.md section 3.13): a real bin (nvBowtie: 0),
 * next_refID = the mate's contig (output_bam.cpp:400 writes a difference of contig indices), NM typed by value (nvBowtie: c, which wraps
 * above 127), paired bits and the mate's placement on unmapped records, no MD:Z:* for an empty MD, TLEN signed on equal begins, no 0x2
 * when a mate was unmapped by the contig rule, and XS from the MAPQ calls' second score (nvBowtie never writes it).
 *
 * Outputs (nvb_bam_out): record i occupies bytes [d_offsets[i], d_offsets[i + 1]) of d_records (16-byte aligned), starting with its
 * block_size; d_offsets[n] is the total size.  d_offsets is always written whole; a record is stored only if it fits whole within
 * `capacity` (d_records may be NULL when capacity is 0: a sizing call).  d_counts[4] = records, mapped, unmapped because the span left
 * its contig or the genome, unmapped because the finish outputs were missing or truncated.
 * NVB_E_INVALID (before any CUDA call) for a NULL in / out / temp_bytes, NULL required pointers (reads, d_n_ops, d_begin, d_strand, the
 * finish arrays, d_score, d_contig_begin, d_names, d_name_offsets, d_offsets, d_counts, d_records with capacity > 0), a misaligned
 * d_records, n_contigs == 0, max_cigar / max_md == 0, 8-bit reads, or an odd n when paired. */
typedef struct nvb_bam_in {
    nvb_string_set   reads;
    const uint8_t*   d_read_quals;     /* may be NULL */
    const uint32_t*  d_n_ops;          /* [n] */
    const nvb_uint2* d_begin;          /* [n] */
    const uint8_t*   d_strand;         /* [n] */
    nvb_finish_out   finish;           /* the outputs of nvb_finish_alignments over the same n alignments */
    const int32_t*   d_score;          /* [n] AS */
    const uint8_t*   d_mapq;           /* [n], may be NULL: MAPQ 255 */
    const int32_t*   d_second_score;   /* [n], may be NULL: no XS */
    const uint32_t*  d_pair_flags;     /* [n / 2] NVB_PAIR_*; NULL: single end */
    const uint32_t*  d_contig_begin;   /* [n_contigs + 1] */
    uint32_t         n_contigs;
    const char*      d_names;
    const uint32_t*  d_name_offsets;   /* [n_names + 1] */
} nvb_bam_in;
typedef struct nvb_bam_out {
    uint8_t*  d_records;
    uint64_t  capacity;
    uint64_t* d_offsets;               /* [n + 1] */
    uint32_t* d_counts;                /* [4] */
} nvb_bam_out;

int nvb_bam_records(const nvb_bam_in* in, uint32_t n, const nvb_bam_out* out, void* d_temp, size_t* temp_bytes, void* stream);

/* BAM records of nvb_seed_extend_all's alignments: several per read.  Same bam1_t encoding, placement and contig rules as nvb_bam_records,
 * single end.  Inputs: base.reads = the n_reads reads (with base.d_read_quals and one name per read); base.d_n_ops / d_begin / d_strand /
 * d_score and base.finish = the per-alignment outputs of nvb_seed_extend_all and of nvb_finish_alignments over its alignment slots (string
 * i of that call's string set is read d_read[i]); base.d_mapq / base.d_second_score are per READ (may be NULL); base.d_pair_flags must be
 * NULL.  d_first / capacity as nvb_seed_extend_all wrote them: read r's alignments are [d_first[r], d_first[r + 1]), stored only if
 * d_first[r + 1] <= capacity.
 * Records, per read in read order: its alignments that pass the placement rule (mapped, span inside one contig), in rank order.  The
 * first is the PRIMARY record: MAPQ d_mapq[r] (255 without it) and XS as in nvb_bam_records; every later one is SECONDARY: FLAG 0x100,
 * MAPQ 255, no XS.  Every mapped record carries NM AS [XS] XM XO XG MD as nvb_bam_records writes them, then NH:i = the read's number of
 * mapped records, typed by htslib's rule.  A read with no placeable alignment -- also one whose range lies beyond capacity -- gets exactly
 * one unmapped record, as nvb_bam_records writes it.  SEQ and QUAL are written in full on every record.  So every read yields exactly one
 * primary or unmapped record.
 * Deliberate deviation from nvBowtie (DESIGN.md section 3.16): it defines SAM_FLAGS_SECONDARY (nvbio/io/output/output_sam.h:57) but never
 * sets it, and writes every all-mode alignment as a primary record with MAPQ 255 (aligner_all.h:83); the SAM specification asks for one
 * primary line per read.
 * Outputs (nvb_bam_out): d_offsets has room for n_reads + capacity + 1 entries; record k = bytes [d_offsets[k], d_offsets[k + 1]) for
 * k < d_counts[0], the number of records (the entries after it repeat the total).  d_counts[1] = mapped records, [2] alignments unmapped
 * by the contig rule, [3] alignments unmapped because finish did not write them whole, plus the reads beyond capacity.  Otherwise the
 * capacity rules of nvb_bam_out.  No host round trip.  NVB_E_INVALID (before any CUDA call) for the checks of nvb_bam_records, a NULL in /
 * d_first, d_pair_flags != NULL, or n_reads + capacity >= 2^31 - 1. */
typedef struct nvb_bam_all_in {
    nvb_bam_in       base;
    const uint32_t*  d_first;          /* [n_reads + 1] */
    uint32_t         capacity;         /* alignment slots of the nvb_seed_extend_all call */
} nvb_bam_all_in;

int nvb_bam_records_all(const nvb_bam_all_in* in, uint32_t n_reads, const nvb_bam_out* out, void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * BGZF compression on the device (SAMv1 section 4.1; the framing of htslib's writer, contrib/htslib/bgzf.c:59 header and
 * bgzf.c:216-240 deflate_block, htslib/bgzf.h:36-37 block sizes; nvBowtie compresses on the host, output_bam.cpp:581-601).
 * Asynchronous on `stream`, no host round trip; NVB_E_TEMP_SIZE protocol.
 *
 * Input: n_bytes bytes at d_in, cut into blocks of exactly 0xFF00 bytes (BGZF_BLOCK_SIZE), the last one possibly shorter; n_blocks =
 * ceil(n_bytes / 0xFF00).  Block i becomes member i, one gzip member (RFC 1952) with the BGZF extra field:
 *   the 18-byte header 1f 8b 08 04 | 00 00 00 00 | 00 ff 06 00 | 'B' 'C' 02 00 | BSIZE = member length - 1 (little-endian);
 *   one raw deflate block (RFC 1951) with BFINAL = 1: dynamic Huffman codes (LZ77 matches up to 258 bytes at distances up to 32768,
 *   code lengths of at most 15 bits, 7 for the code-length code), or a stored block when the dynamic block would not be smaller;
 *   CRC-32 of the block's input, then ISIZE = its length.
 * So no member exceeds 18 + 5 + 65280 + 8 = 65,311 bytes, and each inflates to its block; the members concatenated are a BGZF stream
 * without the 28-byte EOF block, which a file writer appends once.  The output depends only on the input bytes: not on the stream, the
 * grid or timing.
 *
 * Output (nvb_bgzf_out): member i occupies bytes [d_block_offsets[i], d_block_offsets[i + 1]) of d_out; d_block_offsets[n_blocks] is the
 * total.  d_block_offsets is always written whole; a member is stored only if it fits whole within `capacity` (d_out may be NULL when
 * capacity is 0: a sizing call).  A capacity of 65,311 * n_blocks never truncates.
 * NVB_E_INVALID (before any CUDA call) for a NULL out / temp_bytes / d_block_offsets, a NULL d_in with n_bytes > 0, a NULL d_out with
 * capacity > 0, or n_blocks >= 2^32. */
typedef struct nvb_bgzf_out {
    uint8_t*  d_out;
    uint64_t  capacity;
    uint64_t* d_block_offsets;         /* [n_blocks + 1] */
} nvb_bgzf_out;

int nvb_bgzf_compress(const uint8_t* d_in, uint64_t n_bytes, const nvb_bgzf_out* out, void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * Coordinate sort of BAM records on the device.  Asynchronous on `stream`, no host round trip; NVB_E_TEMP_SIZE protocol.
 *
 * Input: n records laid out as nvb_bam_records lays them out, record i = bytes [d_offsets[i], d_offsets[i + 1]) of d_records, starting
 * with its block_size; records may start at any byte offset.
 * Order: key = (refID as uint32, pos as uint32), so unplaced records (refID -1) come last; equal keys keep their input order (a stable
 * sort), so the unplaced records keep their input order too.  This is a valid SO:coordinate order; it does not break ties on the
 * strand as samtools sort does.
 * Output (nvb_bam_sort_out): output record j is input record d_order[j] (d_order may be NULL), at [d_offsets[j], d_offsets[j + 1]) of
 * d_records (16-byte aligned).  d_offsets[n + 1] is always written whole; a record is stored only if it fits whole within `capacity`
 * (d_records may be NULL when capacity is 0).
 * NVB_E_INVALID (before any CUDA call) for a NULL out / temp_bytes / out->d_offsets, a NULL or misaligned out->d_records with capacity
 * > 0, NULL inputs with n > 0, or n >= 2^31 - 1. */
typedef struct nvb_bam_sort_out {
    uint8_t*  d_records;
    uint64_t  capacity;
    uint64_t* d_offsets;               /* [n + 1] */
    uint32_t* d_order;                 /* [n], may be NULL */
} nvb_bam_sort_out;

int nvb_bam_sort(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n, const nvb_bam_sort_out* out, void* d_temp,
                 size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * The BAI index (SAMv1 section 5.2) of a coordinate-sorted, BGZF-compressed BAM file, built on the device.  Asynchronous on `stream`,
 * no host round trip; NVB_E_TEMP_SIZE protocol.  The rules are those of htslib's indexer (contrib/htslib/sam.c:366-424,
 * hts.c:473-696), with the two deviations listed at the end.
 *
 * The file: the header's BGZF members (header_bytes compressed bytes, ending at a member boundary), then nvb_bgzf_compress of exactly
 * d_records[0 : d_offsets[n]] (d_block_offsets is its output), then the 28-byte EOF block.  The records are in nvb_bam_sort order.
 * Virtual offsets are those the reader reports (bgzf_tell), which moves to the next member as soon as it has consumed one: uncompressed
 * byte u < total of the records is ((header_bytes + d_block_offsets[u / 0xFF00]) << 16) | (u % 0xFF00); a record's start is the map of
 * d_offsets[i]; F = (header_bytes + d_block_offsets[n_blocks] + 28) << 16, the file size, ends what no later record ends.
 * Per record: rlen = the sum of the M / D / N / = / X lengths of its CIGAR, 1 when that is 0 (the record's bin field is not read);
 * [beg, end) = [pos, pos + rlen); bin = reg2bin(beg, end) (14 bits, 5 levels), 4680 for an unplaced record; mapped = FLAG lacks 0x4.
 * Chunks, per refID: each maximal run of consecutive records with equal bin gives [start of its first record, start of the next record
 * in the file, or F).  Pseudo-bin 37450 per present refID: (start of its first record, end of its last chunk), (n_mapped, n_unmapped).
 * Bin compression: for levels 5 down to 1, every bin b at that level, its chunks ordered by start: when (last.end >> 16) -
 * (first.start >> 16) < 65536 and the parent (b - 1) >> 3 holds chunks, b's chunks move to the parent and b is dropped.  Then in every
 * real bin a chunk whose start >> 16 <= the previous chunk's end >> 16 joins it.
 * Linear index per refID: n_intv = 1 + max over MAPPED records of (end - 1) >> 14, 0 without a mapped record; entry w = the start of the
 * first mapped record covering window w; a window no record covers takes the refID's first-record start before the first covered
 * window, else the entry before it.
 * Serialisation: "BAI\1", n_ref, per refID n_bin, its bins in ascending bin number (bin, n_chunk, chunks) with the pseudo-bin last,
 * n_intv and the entries; then n_no_coor.
 * Deviations from the htslib of the reference tree (DESIGN.md section 3.15): bins are written in ascending order (htslib: its hash
 * table's order, which the format leaves open), and n_no_coor is the number of unplaced records (htslib stops counting after the first).
 *
 * Output (nvb_bai_out): d_status[0] = 0, or 1 when the records are not in nvb_bam_sort order, 2 when a refID >= n_refs, 3 when a placed
 * record's span leaves [0, 2^29] (the lowest code that applies); d_size[0] = the index's length (0 with a nonzero status); the index is
 * stored only if the status is 0 and it fits whole within `capacity` (d_bai may be NULL when capacity is 0).
 * NVB_E_INVALID (before any CUDA call) for a NULL out / temp_bytes / d_size / d_status / d_offsets / d_block_offsets, a NULL d_bai with
 * capacity > 0, NULL records with n > 0, or n or n_refs >= 2^31 - 1; NVB_E_UNSUPPORTED when max_ref_len > 2^29, which BAI cannot index. */
typedef struct nvb_bai_out {
    uint8_t*  d_bai;
    uint64_t  capacity;
    uint64_t* d_size;                  /* [1] */
    uint32_t* d_status;                /* [1] */
} nvb_bai_out;

int nvb_bam_index(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n, const uint64_t* d_block_offsets, uint64_t header_bytes,
                  uint32_t n_refs, uint32_t max_ref_len, const nvb_bai_out* out, void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * SAM text of BAM records on the device, byte-identical to htslib's sam_format1 (contrib/htslib/sam.c:879-997; nvBowtie's SAM writer,
 * nvbio/io/output/output_sam.cpp).  Asynchronous on `stream`, no host round trip; NVB_E_TEMP_SIZE protocol.
 *
 * Input: n records laid out as nvb_bam_sort accepts them (the outputs of nvb_bam_records, nvb_bam_records_all and nvb_bam_sort as they
 * are): record i = bytes [d_offsets[i], d_offsets[i + 1]) of d_records, starting with its block_size, at any byte offset.  Reference
 * names: bytes d_ref_names, name j = [d_ref_name_offsets[j], d_ref_name_offsets[j + 1]), in the order of the BAM header's reference list.
 * Line i is record i formatted as sam_format1 formats it, then '\n':
 *   QNAME (l_read_name - 1 bytes), FLAG;  RNAME, '*' for refID -1;  POS + 1 (an unplaced record prints 0);  MAPQ;
 *   CIGAR as <len><op> over "MIDNSHP=X", '*' without ops;  RNEXT: '*' for next_refID -1, '=' when it equals refID, else the name;
 *   PNEXT + 1;  TLEN signed;  SEQ in "=ACMGRSVTWYHKDBN" and QUAL + 33 ('*' when the first QUAL byte is 0xFF), "*\t*" when l_seq is 0;
 *   the tags in record order, "\tXX:i:<v>" for types c C s S i I (I unsigned) and "\tXX:Z:<s>" for Z.
 * Integers are printed in decimal as 32-bit values (POS + 1 and PNEXT + 1 wrap as htslib's int arithmetic does), fields separated by one
 * TAB.  A record is REJECTED and gets a line of 0 bytes when: block_size + 4 is not its extent; its fixed fields, name, CIGAR, SEQ, QUAL or
 * a tag run past its end; its name is empty (l_read_name < 2) or not NUL-terminated; refID or next_refID lies outside [-1, n_refs); a CIGAR
 * op is above 8; a tag type is not one of c C s S i I Z, or a Z value has no NUL; or 1-3 bytes are left after its last tag.
 * (Tag types A f d H B are never written by this library's record writers and are not formatted.)
 *
 * Output (nvb_sam_out): line i occupies bytes [d_offsets[i], d_offsets[i + 1]) of d_text, '\n' included; d_offsets[n] is the total.
 * d_offsets is always written whole; a line is stored only if it fits whole within `capacity`, so the stored lines are a prefix (d_text
 * may be NULL when capacity is 0: a sizing call).  d_rejected[0] = rejected records, d_rejected[1] = the index of the first, 0xFFFFFFFF
 * when none.  n = 0 writes d_offsets[0] = 0 and d_rejected = (0, 0xFFFFFFFF).
 * NVB_E_INVALID (before any CUDA call) for a NULL out / temp_bytes / d_offsets / d_rejected, a NULL d_text with capacity > 0, NULL records
 * with n > 0, NULL names with n_refs > 0, or n >= 2^31 - 1. */
typedef struct nvb_sam_out {
    char*     d_text;
    uint64_t  capacity;
    uint64_t* d_offsets;               /* [n + 1] */
    uint32_t* d_rejected;              /* [2] */
} nvb_sam_out;

int nvb_sam_format(const uint8_t* d_records, const uint64_t* d_offsets, uint32_t n,
                   const char* d_ref_names, const uint32_t* d_ref_name_offsets, uint32_t n_refs,
                   const nvb_sam_out* out, void* d_temp, size_t* temp_bytes, void* stream);

/* -------------------------------------------------------------------------------------------
 * Host-buffer entry point: batches of reads in HOST memory in, per-read results in HOST memory out.
 * Replaces nvBowtie's input thread -> compute thread hand-off and its per-stage cudaDeviceSynchronize
 * (nvBowtie/bowtie2/cuda/compute_thread.cu:213-243, nvBowtie/bowtie2/cuda/defs.h:64, aligner_best_approx.h:219-241):
 * `depth` batches are in flight at once -- the host->device copy of batch i+1 and the device->host copy of batch i-1
 * overlap the kernels of batch i on separate streams.  By default all batches share ONE compute stream (their kernels run back
 * to back); the environment variable NVB_PIPELINE_COMPUTE_STREAMS=k (read at creation) spreads consecutive batches over k
 * compute streams so that kernels of neighbouring batches may share the SMs.
 *
 * Reads: n_reads fixed-stride strings of `read_len` symbols, `words_per_read` 32-bit words each (big-endian packing,
 * read_bits = 2 or 4).  pair_params != NULL: paired-end (reads = mate 1 of every pair, then mate 2; n_reads even).
 * submit() takes a host pointer (pinned memory makes the copy asynchronous) that must stay valid until wait() returns for
 * that ticket; wait() blocks until that batch's results are in the pipeline's own pinned host buffers and returns pointers
 * to them (valid until `depth` further batches have been submitted).  One pipeline is used from one host thread.
 * ------------------------------------------------------------------------------------------- */
typedef struct nvb_pipeline nvb_pipeline;
typedef struct nvb_pipeline_result {
    const int32_t*  best_score;    /* [n_reads]  single end (NULL when paired) */
    const uint32_t* best_pos;      /* [n_reads]  */
    const uint32_t* n_hits;        /* [3] hits kept, found, distinct alignment jobs */
    const int32_t*  pair_score;    /* [n_pairs]   paired end (NULL when single end), as nvb_pair_out */
    const uint32_t* pair_flags;    /* [n_pairs]   */
    const int32_t*  mate_score;    /* [2*n_pairs] */
    const uint32_t* mate_pos;      /* [2*n_pairs] */
    const uint8_t*  mate_strand;   /* [2*n_pairs] */
    const uint32_t* n_rescue;      /* [2] */
    float           device_ms;     /* device time of this batch's kernels (its compute stream), for reporting */
} nvb_pipeline_result;

int  nvb_pipeline_create(const nvb_fm_index* fmi, const uint32_t* d_genome, const nvb_seed_extend_params* params,
                         const nvb_pair_params* pair_params /* NULL = single end */,
                         uint32_t n_reads, uint32_t read_len, uint32_t words_per_read, uint32_t read_bits,
                         uint32_t hit_capacity, uint32_t depth, nvb_pipeline** out);
int  nvb_pipeline_submit(nvb_pipeline* p, const uint32_t* h_read_words, uint32_t* ticket);
int  nvb_pipeline_wait(nvb_pipeline* p, uint32_t ticket, nvb_pipeline_result* out);
/* bytes moved per batch: host -> device, device -> host (a BAM pipeline: the largest input of a batch, and the fixed part of its results;
   the payload adds its own byte count) */
void nvb_pipeline_traffic(const nvb_pipeline* p, size_t* h2d_bytes, size_t* d2h_bytes);
void nvb_pipeline_destroy(nvb_pipeline* p);

/* BAM mode of the pipeline: host reads, qualities and names in, the batch's BAM payload out (nvBowtie's input thread -> compute thread ->
 * output writer, compute_thread.cu:213-243, output_bam.cpp:581-601).  Same slots, streams, events, depth and NVB_PIPELINE_COMPUTE_STREAMS
 * rules as above; one batch runs on its slot's compute stream, each call with its own rules unchanged:
 *   single end: nvb_seed_extend_mapq with best_alignment -> nvb_finish_alignments -> nvb_bam_records, one name per read;
 *   paired:     nvb_seed_extend_paired_traceback with mapq (every policy and flag, NVB_PE_DISCORDANT included) -> nvb_finish_alignments
 *               over the 2n mates with d_strand = d_mate_strand -> nvb_bam_records with d_pair_flags, one name per pair;
 *   then, with compress, the BGZF members of exactly the d_offsets[n] record bytes (nvb_bgzf_compress's output for them, with the byte
 *   count read on the device: no host round trip inside a batch).
 * Genome length for finish: fmi->length.  MAPQ and XS of the records come from the mapping call; qualities go to the mapping call
 * (params.d_read_quals) and to the records.
 *
 * submit: n_reads (1 .. max_reads; even when paired: mate 1 of every pair, then mate 2, so a short last batch is fine) reads of
 * words_per_read words; h_quals (has_quals): one byte per read symbol, n_reads * words_per_read * (32 / read_bits) bytes in the layout of
 * the symbols; h_lengths (has_lengths): per-read lengths 1 .. read_len, else every read is read_len long; names: h_names bytes and
 * h_name_offsets[n_names + 1] (n_names = n_reads, or n_reads / 2 when paired), offsets from 0, each name 1 or more bytes (names longer
 * than 254 bytes are cut, as nvb_bam_records does), the last offset <= max_name_bytes.  As in nvb_pipeline_submit, host buffers must
 * stay valid until wait returns for that ticket (pinned memory makes the copies asynchronous).
 * wait: nvb_pipeline_bam_result, pointers into the slot's pinned host memory, valid until `depth` further submits.  The counts leave the
 * device with the batch; the payload is then copied with exactly its byte count (by wait, or by the submit that reuses a slot whose
 * batch was never waited for).  The host payload buffer of a slot grows (cudaHostAlloc) to the largest payload it has held.
 * payload: with compress, BGZF members that a BAM writer emits verbatim between the header and the EOF block; without, the record stream.
 *
 * Slot memory: one device allocation per slot (nvb_pipeline_slot_bytes).  Buffers whose lifetimes do not overlap share bytes: the
 * mapping call's temp (direction matrices included) is dead once finish starts, the traceback ops once the records are built, the finish
 * outputs once the records exist, the records once BGZF's first kernel has read them (its members are written over them).  With n =
 * max_reads, L = read_len: O = n * max_ops (ops), T = the mapping call's temp, F = n * (4 * max_cigar + max_md + 28) (finish outputs),
 * B = the records' temp, R = n * (36 + 1 + 4 * max_cigar + (L + 1) / 2 + L + 46 + max_md) + max_name_bytes (twice when paired) (the
 * record bound), Zo = 65,311 * ceil(R / 0xFF00) (members), Zt = the BGZF temp (about R, + 17 MB on an H100): the stage region takes
 * max(O + T, max(O, R) + F + B, max(R, Zo) + Zt) bytes with compress and max(O + T, max(O, R) + F + B) without, beside O(n) bytes of
 * inputs and per-read outputs.  From shapes, not measured: 1 M mates of 150 bp, band 31, default sizes: O 0.33 GB, F 2.4 GB, R 2.6 GB.
 *
 * NVB_E_INVALID before any CUDA call: the checks of nvb_pipeline_create (bar its refusal of NVB_PE_DISCORDANT); bam, mapq, d_min_score
 * or d_contig_begin NULL, n_contigs == 0, max_name_bytes == 0; params->d_read_quals != NULL (qualities come per batch); a quality table
 * without has_quals; mapq->max_read_len < read_len.  In submit: n_reads == 0 or > max_reads, odd when paired; a NULL array the flags
 * require (words, names, offsets, ticket; quals with has_quals; lengths with has_lengths); name offsets that do not start at 0, do not
 * increase, or end past max_name_bytes; a length of 0 or above read_len.  submit / wait of the other kind of pipeline.
 * NVB_E_UNSUPPORTED for read_len > 512 (the traceback calls' limit). */
typedef struct nvb_pipeline_bam_params {
    const nvb_mapq_params* mapq;          /* required: d_min_score, max_read_len >= read_len, match_bonus */
    const uint32_t* d_contig_begin;       /* [n_contigs + 1], as nvb_bam_in */
    uint32_t        n_contigs;
    uint32_t        max_name_bytes;       /* bytes of names per batch */
    uint32_t        has_quals;            /* 1: every submit passes qualities */
    uint32_t        has_lengths;          /* 1: every submit passes per-read lengths (<= read_len) */
    uint32_t        compress;             /* 1: BGZF members; 0: the raw record stream */
    uint32_t        max_ops, max_cigar, max_md;   /* 0 = never truncate: 2 * read_len + band_len, max_ops + 2, 3 * max_ops + 1 */
} nvb_pipeline_bam_params;
typedef struct nvb_pipeline_bam_result {
    const uint8_t*  payload;         /* BGZF members (compress) or BAM records */
    uint64_t        payload_bytes;
    uint64_t        record_bytes;    /* bytes of the records (= payload_bytes without compress) */
    uint32_t        n_records;       /* 2 per pair when paired */
    uint32_t        n_blocks;        /* BGZF members (0 without compress) */
    const uint32_t* counts;          /* [4] nvb_bam_records' tallies: records, mapped, unmapped by the contig rule, unfinished */
    const uint32_t* n_hits;          /* [3] hits kept, found, distinct alignment jobs */
    const uint32_t* n_rescue;        /* [2] paired (NULL when single end): full-DP jobs run, wanted */
    float           device_ms;       /* device time of this batch's kernels (its compute stream) */
} nvb_pipeline_bam_result;

int  nvb_pipeline_create_bam(const nvb_fm_index* fmi, const uint32_t* d_genome, const nvb_seed_extend_params* params,
                             const nvb_pair_params* pair_params /* NULL = single end */, const nvb_pipeline_bam_params* bam,
                             uint32_t max_reads, uint32_t read_len, uint32_t words_per_read, uint32_t read_bits,
                             uint32_t hit_capacity, uint32_t depth, nvb_pipeline** out);
int  nvb_pipeline_submit_bam(nvb_pipeline* p, uint32_t n_reads, const uint32_t* h_read_words, const uint8_t* h_quals,
                             const uint32_t* h_lengths, const char* h_names, const uint32_t* h_name_offsets, uint32_t* ticket);
int  nvb_pipeline_wait_bam(nvb_pipeline* p, uint32_t ticket, nvb_pipeline_bam_result* out);
/* bytes of device memory one slot of a BAM pipeline holds (its single allocation) */
size_t nvb_pipeline_slot_bytes(const nvb_pipeline* p);

/* Profiling aid (the reference wraps every stage in cuda::Timer, nvBowtie/bowtie2/cuda/aligner_best_approx.h:
 * 219-241): device time in ms of the seven stages of the most recent nvb_seed_extend call -- [fw,rc] strings,
 * seed match (FM-index), hit slots, locate + windows, job de-duplication, banded extension, best-per-read (which includes the
 * traceback and, in nvb_seed_extend_mapq / nvb_seed_extend_paired_mapq, the second-best passes and the MAPQ).  Synchronises on the
 * call's last event. */
int nvb_seed_extend_stage_ms(float ms[7]);

#ifdef __cplusplus
}
#endif
#endif /* NVBIO_B200_H */
