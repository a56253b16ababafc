/* oracle/nvb_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded restatement of the reference algorithms on the two hot paths of
 * NVlabs/nvbio (citations are relative to /root/reference).  It exists so that the CUDA path can
 * be checked on the GPU box, where /root/reference does not exist.  It is PINNED: tests/test_oracle.py
 * checks every function here against (a) the reference's own templates compiled unmodified into
 * oracle/_ref/libnvbio_ref.so (oracle/ref_shim.cpp), (b) the golden vectors of the reference's tests
 * (nvbio-test/alignment_test.cu:761-825, fmindex/bwt.h:81-86) committed under tests/golden/.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  The product (nvbio_b200/) never links or calls it.
 *
 * Build: make -C oracle   (gcc -O2 -shared -fPIC)
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <limits.h>

typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t  i32;
typedef uint8_t  u8;

/* ------------------------------------------------------------------------------------------------
 * 2-bit big-endian packed streams: symbol i lives in word i>>4 at bit shift 30-2*(i&15)
 * (nvbio/basic/packedstream_inl.h:336-372, PackedStream<...,2,true>)
 * ---------------------------------------------------------------------------------------------- */
static inline u32 get2be(const u32* w, u64 i) { return (w[i >> 4] >> (30u - 2u*(u32)(i & 15u))) & 3u; }
static inline void set2be(u32* w, u64 i, u32 c)
{
    const u32 sh = 30u - 2u*(u32)(i & 15u);
    w[i >> 4] = (w[i >> 4] & ~(3u << sh)) | ((c & 3u) << sh);
}

void orc_pack2be(u32 n, const u8* sym, u32* words) /* words must hold ceil(n/16), pre-zeroed or not */
{
    const u32 nw = (n + 15u) / 16u;
    memset(words, 0, sizeof(u32) * nw);
    for (u32 i = 0; i < n; ++i) set2be(words, i, sym[i]);
}

/* ------------------------------------------------------------------------------------------------
 * Suffix array / BWT / SSA (semantics of nvbio/fmindex/bwt.h:38-63: SA has n+1 entries, SA[0]=n is
 * the empty suffix `$`; BWT row r holds T[SA[r]-1]; the `$` row (primary) is removed from the BWT).
 * The construction here is a plain prefix-doubling sort -- independent of contrib/sais.h.
 * ---------------------------------------------------------------------------------------------- */
static const u32* g_rank; static u32 g_h; static u32 g_n;
static int cmp_sfx(const void* a, const void* b)
{
    const u32 i = *(const u32*)a, j = *(const u32*)b;
    if (g_rank[i] != g_rank[j]) return g_rank[i] < g_rank[j] ? -1 : 1;
    /* rank of the suffix h further on; the empty suffix (position n) ranks lowest (0) */
    const u32 ri = (i + g_h <= g_n) ? g_rank[i + g_h] : 0u;
    const u32 rj = (j + g_h <= g_n) ? g_rank[j + g_h] : 0u;
    if (ri != rj) return ri < rj ? -1 : 1;
    return 0;
}

/* sa: n+1 entries out.  text: n unpacked symbols (0..3) */
void orc_suffix_array(u32 n, const u8* text, i32* sa_out)
{
    u32* sa   = (u32*)malloc(sizeof(u32) * (n + 1));
    u32* rank = (u32*)malloc(sizeof(u32) * (n + 2));
    u32* tmp  = (u32*)malloc(sizeof(u32) * (n + 2));
    for (u32 i = 0; i <= n; ++i) { sa[i] = i; rank[i] = (i < n) ? 1u + text[i] : 0u; }
    rank[n + 1] = 0;
    g_n = n;
    for (u32 h = 1;; h *= 2)
    {
        g_rank = rank; g_h = h;
        qsort(sa, n + 1, sizeof(u32), cmp_sfx);
        tmp[sa[0]] = 0;
        u32 distinct = 1;
        for (u32 k = 1; k <= n; ++k)
        {
            if (cmp_sfx(&sa[k - 1], &sa[k]) != 0) ++distinct;
            tmp[sa[k]] = distinct - 1;
        }
        memcpy(rank, tmp, sizeof(u32) * (n + 1));
        if (distinct == n + 1 || h > n) break;
    }
    for (u32 k = 0; k <= n; ++k) sa_out[k] = (i32)sa[k];
    free(sa); free(rank); free(tmp);
}

/* bwt: packed 2-bit big-endian, bwt_words words (zeroed here).  returns primary.
 * (nvbio/fmindex/bwt.h:51-63) */
u32 orc_bwt_from_sa(u32 n, const u8* text, const i32* sa, u32* bwt, u32 bwt_words)
{
    memset(bwt, 0, sizeof(u32) * bwt_words);
    u32 primary = 0, out = 0;
    for (u32 r = 0; r <= n; ++r)
    {
        if (sa[r] == 0) { primary = r; continue; }
        set2be(bwt, out++, text[sa[r] - 1]);
    }
    return primary;
}

/* occ[k*4+c] = #c in bwt[0,64k), k < ceil(n/64); cnt[c] totals
 * (nvbio/fmindex/rank_dictionary_inl.h:42-77) */
void orc_build_occ(u32 n, const u32* bwt, u32* occ, u32* cnt)
{
    u32 counters[4] = {0, 0, 0, 0};
    for (u32 i = 0; i < n; ++i)
    {
        if ((i & 63u) == 0) for (u32 c = 0; c < 4; ++c) occ[(i / 64u) * 4u + c] = counters[c];
        ++counters[get2be(bwt, i)];
    }
    for (u32 c = 0; c < 4; ++c) cnt[c] = counters[c];
}

/* block k (32 bytes) = {4 BWT words, occ[A,C,G,T]} (nvbio/io/fmindex/fmindex_impl.cu:308-322);
 * L2 = exclusive prefix sums of cnt (:324-327).  seq_words must be a multiple of 4. */
void orc_interleave(u32 seq_words, const u32* bwt, const u32* occ, const u32* cnt, u32* bwt_occ, u32* L2)
{
    for (u32 w = 0; w < seq_words; w += 4)
    {
        for (u32 q = 0; q < 4; ++q) bwt_occ[w * 2 + q]     = bwt[w + q];
        for (u32 q = 0; q < 4; ++q) bwt_occ[w * 2 + 4 + q] = occ[w + q];
    }
    L2[0] = 0;
    for (u32 c = 0; c < 4; ++c) L2[c + 1] = L2[c] + cnt[c];
}

/* ssa[r/16] = SA[r] for r % 16 == 0; ssa[0] = -1  (nvbio/fmindex/ssa_inl.h:262-277,
 * nvbio/io/fmindex/fmindex_impl.cu:244) */
void orc_build_ssa(u32 n, const i32* sa, u32* ssa)
{
    const u32 n_items = (n + 16u) / 16u;
    for (u32 i = 0; i < n_items; ++i) ssa[i] = (u32)sa[i * 16u];
    ssa[0] = 0xFFFFFFFFu;
}

/* count table known answer (nvbio/fmindex/bwt.h:81-98) */
void orc_count_table(u32* t)
{
    for (u32 i = 0; i < 256; ++i)
    {
        u32 x = 0;
        for (u32 j = 0; j < 4; ++j)
            x |= (u32)(((i & 3) == j) + ((i >> 2 & 3) == j) + ((i >> 4 & 3) == j) + ((i >> 6) == j)) << (j << 3);
        t[i] = x;
    }
}

/* ------------------------------------------------------------------------------------------------
 * rank dictionary over the interleaved layout (nvbio/fmindex/rank_dictionary_inl.h:424-538,
 * nvbio/basic/popcount_inl.h:239-247, 327-350)
 * ---------------------------------------------------------------------------------------------- */
static inline u32 popc32(u32 x) { return (u32)__builtin_popcount(x); }
static inline u32 popc2bit(u32 w, u32 c)
{
    const u32 odd  = ((c & 2u) ? w : ~w) >> 1;
    const u32 even = ((c & 1u) ? w : ~w);
    return popc32(odd & even & 0x55555555u);
}
/* count of c among symbols 0..r (inclusive) of word w: zero the low 2t bits (t = 15-r) and, for c==0,
 * subtract the t spurious zeros */
static inline u32 popc2bit_upto(u32 w, u32 c, u32 r)
{
    const u32 t = 15u - r;
    const u32 m = w & ~((1u << (2u * t)) - 1u);
    return popc2bit(m, c) - (c == 0 ? t : 0u);
}

u32 orc_dict_rank(const u32* bwt_occ, u32 i, u32 c)
{
    if (i == 0xFFFFFFFFu) return 0;
    const u32 k = i >> 6, m = (i & 63u) >> 4;
    const u32* blk = bwt_occ + (u64)k * 8u;
    u32 x = blk[4 + c];
    for (u32 q = 0; q < m; ++q) x += popc2bit(blk[q], c);
    return x + popc2bit_upto(blk[m], c, i & 15u);
}

typedef struct { const u32* bwt_occ; const u32* ssa; u32 n; u32 primary; u32 L2[5]; } orc_index;

/* fm_index-level rank with `$` handling (nvbio/fmindex/fmindex_inl.h:36-57) */
static u32 fm_rank1(const orc_index* f, u32 k, u32 c)
{
    if (k == 0xFFFFFFFFu) return 0;
    if (k == f->n) return f->L2[c + 1] - f->L2[c];
    if (k >= f->primary) --k;
    return orc_dict_rank(f->bwt_occ, k, c);
}

/* range form (nvbio/fmindex/fmindex_inl.h:66-99 -> rank_dictionary_inl.h:500-523); also counts the
 * distinct 32-byte blocks that must be fetched (SURVEY.md 8d) */
static void fm_rank2(const orc_index* f, u32 x, u32 y, u32 c, u32* rx, u32* ry, u64* blocks)
{
    if (x == y) { *rx = *ry = fm_rank1(f, x, c); if (blocks && x != 0xFFFFFFFFu && x != f->n) ++*blocks; return; }
    if (x == 0xFFFFFFFFu) { *rx = 0; *ry = fm_rank1(f, y, c); if (blocks && y != f->n) ++*blocks; return; }
    if (y == f->n) { *rx = fm_rank1(f, x, c); *ry = f->L2[c + 1] - f->L2[c]; if (blocks) ++*blocks; return; }
    if (x >= f->primary) --x;
    if (y >= f->primary) --y;
    /* dictionary level */
    if (x == 0xFFFFFFFFu && y == 0xFFFFFFFFu) { *rx = *ry = 0; return; }
    if (x == 0xFFFFFFFFu || x == y)
    {
        const u32 r = orc_dict_rank(f->bwt_occ, y, c);
        *rx = (x == 0xFFFFFFFFu) ? 0u : r; *ry = r;
        if (blocks) ++*blocks;
        return;
    }
    *rx = orc_dict_rank(f->bwt_occ, x, c);
    *ry = orc_dict_rank(f->bwt_occ, y, c);
    if (blocks) *blocks += ((x >> 6) == (y >> 6)) ? 1u : 2u;
}

void orc_rank(const u32* bwt_occ, const u32* L2, u32 n, u32 primary, const u32* k, const u8* c, u32 nq, u32* out)
{
    orc_index f = { bwt_occ, NULL, n, primary, { L2[0], L2[1], L2[2], L2[3], L2[4] } };
    for (u32 i = 0; i < nq; ++i) out[i] = fm_rank1(&f, k[i], c[i]);
}

/* backward search, nvBowtie's form: a symbol > 3 aborts with the empty range (1,0)
 * (nvbio/fmindex/fmindex_inl.h:307-341; nvBowtie/bowtie2/cuda/mapping_inl.h:83-97).
 * Queries are unpacked symbols.  Returns the total number of 32-byte blocks touched. */
/* blocks_from_step: LF steps with index < blocks_from_step are not counted in the returned block total
 * (used to size the traffic of a search whose first k steps are replaced by a k-mer table look-up) */
u64 orc_match_from(const u32* bwt_occ, const u32* L2, u32 n, u32 primary,
              const u8* q, const u32* off, const u32* len, u32 nq, u32* out_xy, u32 blocks_from_step)
{
    orc_index f = { bwt_occ, NULL, n, primary, { L2[0], L2[1], L2[2], L2[3], L2[4] } };
    u64 blocks = 0, skipped = 0;
    for (u32 s = 0; s < nq; ++s)
    {
        u32 x = 0, y = n;
        const u8* p = q + off[s];
        u32 step = 0;
        for (i32 i = (i32)len[s] - 1; i >= 0 && x <= y; --i, ++step)
        {
            const u32 c = p[i];
            if (c > 3) { x = 1; y = 0; break; }
            u32 rx, ry;
            fm_rank2(&f, x - 1u, y, c, &rx, &ry, step >= blocks_from_step ? &blocks : &skipped);
            x = f.L2[c] + rx + 1u;
            y = f.L2[c] + ry;
        }
        out_xy[2 * s] = x; out_xy[2 * s + 1] = y;
    }
    return blocks;
}
u64 orc_match(const u32* bwt_occ, const u32* L2, u32 n, u32 primary,
              const u8* q, const u32* off, const u32* len, u32 nq, u32* out_xy)
{
    return orc_match_from(bwt_occ, L2, n, primary, q, off, len, nq, out_xy, 0);
}

/* locate: LF-walk to the next sampled row (rows that are multiples of 16), then ssa + steps
 * (nvbio/fmindex/fmindex_inl.h:471-499, ssa_inl.h:487-504).  Returns total LF steps. */
u64 orc_locate(const u32* bwt_occ, const u32* ssa, const u32* L2, u32 n, u32 primary,
               const u32* rows, u32 nq, u32* out)
{
    orc_index f = { bwt_occ, ssa, n, primary, { L2[0], L2[1], L2[2], L2[3], L2[4] } };
    u64 steps = 0;
    for (u32 s = 0; s < nq; ++s)
    {
        u32 j = rows[s], t = 0;
        while ((j & 15u) != 0)
        {
            if (j != primary)
            {
                const u32 k = j < primary ? j : j - 1u;
                const u32 c = (bwt_occ[(u64)(k >> 6) * 8u + ((k & 63u) >> 4)] >> (30u - 2u * (k & 15u))) & 3u;
                j = f.L2[c] + fm_rank1(&f, j, c);
            }
            else j = 0;
            ++t;
        }
        steps += t;
        out[s] = ssa[j >> 4] + t;
    }
    return steps;
}

/* ------------------------------------------------------------------------------------------------
 * banded Gotoh score (nvbio/alignment/gotoh/gotoh_banded_inl.h:406-658, init :46-77; sink
 * nvbio/alignment/sink_inl.h:39-65; text cache nvbio/alignment/alignment_base_inl.h:75-99).
 *
 * type: 0 GLOBAL, 1 LOCAL, 2 SEMI_GLOBAL.  Substitution score: qtab == NULL -> (r==q ? match : mismatch)
 * (SimpleGotohScheme, nvbio/alignment/utils.h:114-135); else (r==q ? qtab[2*qq] : qtab[2*qq+1])
 * (nvBowtie SmithWatermanScoringScheme::substitution, nvBowtie/bowtie2/cuda/scoring.h:281).
 * E and F both use the PATTERN gap costs (gotoh_banded_inl.h:444-445); the text gap costs only enter
 * the GLOBAL row-0 initialisation and the infimum.
 * Patterns / texts are unpacked 8-bit symbols.  For BAND not in {3,5,7,15} the sliding text cache is
 * 2-bit packed, so cached symbols are masked to 2 bits while the freshly fetched one (cell B-1) is not.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    i32 match, mismatch;
    i32 pattern_gap_open, pattern_gap_ext, text_gap_open, text_gap_ext;
} orc_scheme;

static inline i32 imax(i32 a, i32 b) { return a > b ? a : b; }

#define ORC_MAX_BAND 64
/* score of a sink that received no report: Field_traits<int32>::min() (nvbio/basic/numbers.h:832-836) */
#define ORC_SINK_MIN (-(1 << 30))

/* optional aln::Best2Sink<int32> fed with the same reports (nvbio/alignment/sink.h:114-147, sink_inl.h:70-116): when set, every
 * report() of the DP also reaches it */
typedef struct { i32 s1, s2; u32 x1, y1, x2, y2, dist; } orc_best2;
static orc_best2* g_best2 = NULL;
static inline void best2_report(orc_best2* b, i32 s, u32 x, u32 y)
{
    if (b->s1 <= s) { b->s1 = s; b->x1 = x; b->y1 = y; }
    else if (b->s2 <= s && (x + b->dist < b->x1 || x > b->x1 + b->dist)) { b->s2 = s; b->x2 = x; b->y2 = y; }
}
static inline void sink_report(i32* best, u32* bx, u32* by, i32 s, u32 x, u32 y)
{
    if (*best <= s) { *best = s; *bx = x; *by = y; }
    if (g_best2) best2_report(g_best2, s, x, y);
}

/* returns 1 when scored, 0 when text_len < pattern_len (score/sink left at BestSink defaults) */
int orc_banded_gotoh_one(int B, int type, const orc_scheme* S, const i32* qtab,
                         const u8* P, const u8* Q, u32 M, const u8* T, u32 N,
                         i32* out_score, u32* out_x, u32* out_y)
{
    i32 best = ORC_SINK_MIN; u32 bx = 0xFFFFFFFFu, by = 0xFFFFFFFFu;
    *out_score = best; *out_x = bx; *out_y = by;
    if (N < M) return 0;

    const int packed_cache = !(B == 3 || B == 5 || B == 7 || B == 15);
    const i32 Go = S->pattern_gap_open, Ge = S->pattern_gap_ext;
    const i32 INF = SHRT_MIN - imax(imax(Go, Ge), imax(S->text_gap_open, S->text_gap_ext));

    i32 H[ORC_MAX_BAND], F[ORC_MAX_BAND];
    u32 cache[ORC_MAX_BAND];
    H[0] = 0;
    for (int j = 1; j < B; ++j) H[j] = (type == 0) ? S->text_gap_open + (j - 1) * S->text_gap_ext : 0;
    for (int j = 0; j < B; ++j) F[j] = INF;
    /* the reference reads text[j] for j < B-1 without a bound check; positions >= N are undefined there.
       We define them as 255 (then masked like any cached symbol). */
    for (int j = 0; j < B - 1; ++j) { const u32 g = ((u32)j < N) ? T[j] : 255u; cache[j] = packed_cache ? (g & 3u) : g; }

#define SUB(g, q, qq) (qtab ? (((u8)(g) == (q)) ? qtab[2 * (qq)] : qtab[2 * (qq) + 1]) : (((u8)(g) == (q)) ? S->match : S->mismatch))

    for (u32 i = 0; i < M; ++i)
    {
        const u8 q = P[i];
        const u8 qq = Q ? Q[i] : 0;
        /* j = 0 */
        {
            F[0] = imax(F[1] + Ge, H[1] + Go);
            const u32 g = cache[0];
            i32 h = imax(F[0], H[0] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + 1, i + 1); }
            H[0] = h;
        }
        i32 E = H[0] + Go;
        for (int j = 1; j < B - 1; ++j)
        {
            F[j] = imax(F[j + 1] + Ge, H[j + 1] + Go);
            const u32 g = cache[j]; cache[j - 1] = g;
            i32 h = imax(imax(F[j], E), H[j] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + (u32)j + 1, i + 1); }
            H[j] = h;
            E = imax(h + Go, E + Ge);
        }
        const u8 g = (i + (u32)B - 1 < N) ? T[i + B - 1] : 255u;
        cache[B - 2] = packed_cache ? (g & 3u) : g;
        {
            F[B - 1] = INF;
            i32 h = imax(E, H[B - 1] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + (u32)B, i + 1); }
            H[B - 1] = h;
        }
    }
#undef SUB
    if (type == 0) sink_report(&best, &bx, &by, H[B - 1], M + (u32)B - 1, M);
    else if (type == 2)
    {
        const u32 lim = (M + (u32)B - 1 < N ? M + (u32)B - 1 : N) - (M - 1);
        sink_report(&best, &bx, &by, H[0], M, M);
        for (int j = 1; j < B; ++j) if ((u32)j < lim) sink_report(&best, &bx, &by, H[j], M + (u32)j, M);
    }
    *out_score = best; *out_x = bx; *out_y = by;
    return 1;
}

void orc_banded_gotoh(int B, int type, const orc_scheme* S, const i32* qtab,
                      const u8* pat, const u8* qual, const u32* p_off, const u32* p_len,
                      const u8* txt, const u32* t_off, const u32* t_len,
                      u32 n, i32* score, u32* sink_x, u32* sink_y, u8* ok)
{
    for (u32 i = 0; i < n; ++i)
    {
        const int r = orc_banded_gotoh_one(B, type, S, qtab,
            pat + p_off[i], qual ? qual + p_off[i] : NULL, p_len[i],
            txt + t_off[i], t_len[i], &score[i], &sink_x[i], &sink_y[i]);
        if (ok) ok[i] = (u8)r;
    }
}

/* banded Gotoh with a Best2Sink: out6[i] = (score1, sink1.x, sink1.y, score2, sink2.x, sink2.y) as int64 */
void orc_banded_gotoh_best2(int B, int type, const orc_scheme* S, const u8* pat, const u32* p_off, const u32* p_len,
                            const u8* txt, const u32* t_off, const u32* t_len, u32 n, u32 distinct_dist, long long* out6)
{
    for (u32 i = 0; i < n; ++i)
    {
        orc_best2 b = { ORC_SINK_MIN, ORC_SINK_MIN, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, distinct_dist };
        i32 sc; u32 x, y;
        g_best2 = &b;
        orc_banded_gotoh_one(B, type, S, NULL, pat + p_off[i], NULL, p_len[i], txt + t_off[i], t_len[i], &sc, &x, &y);
        g_best2 = NULL;
        long long* o = out6 + 6 * (size_t)i;
        o[0] = b.s1; o[1] = b.x1; o[2] = b.y1; o[3] = b.s2; o[4] = b.x2; o[5] = b.y2;
    }
}

/* ------------------------------------------------------------------------------------------------
 * windowed banded Gotoh score: aln::banded_alignment_score<B>(aligner, pattern, quals, text, min_score, window_begin, window_end,
 * sink, checkpoint) (nvbio/alignment/banded_inl.h:178-218 -> gotoh_banded_inl.h:706-739 with GotohCheckpointedScoringContext
 * :132-199): rows [wb, we) of the band only; wb > 0 starts from the checkpoint (H,F as short2 per band cell), every call stores
 * the checkpoint of row `we` clamped at SHRT_MIN+32; when rows remain the call returns 0 if the band maximum can no longer
 * reach min_score (:616-634); the final reports happen when we == M.  `best/bx/by` are the caller's BestSink (in/out).
 * ---------------------------------------------------------------------------------------------- */
int orc_banded_gotoh_window_one(int B, int type, const orc_scheme* S, const i32* qtab,
                                const u8* P, const u8* Q, u32 M, const u8* T, u32 N, u32 wb, u32 we, i32 min_score,
                                short* ckpt, i32* best_io, u32* bx_io, u32* by_io)
{
    i32 best = *best_io; u32 bx = *bx_io, by = *by_io;
    if (N < M) return 0;
    const int packed_cache = !(B == 3 || B == 5 || B == 7 || B == 15);
    const i32 Go = S->pattern_gap_open, Ge = S->pattern_gap_ext;
    const i32 INF = SHRT_MIN - imax(imax(Go, Ge), imax(S->text_gap_open, S->text_gap_ext));
    i32 H[ORC_MAX_BAND], F[ORC_MAX_BAND]; u32 cache[ORC_MAX_BAND];
    if (wb == 0)
    {
        H[0] = 0;
        for (int j = 1; j < B; ++j) H[j] = (type == 0) ? S->text_gap_open + (j - 1) * S->text_gap_ext : 0;
        for (int j = 0; j < B; ++j) F[j] = INF;
    }
    else for (int j = 0; j < B; ++j) { H[j] = ckpt[2 * j]; F[j] = ckpt[2 * j + 1]; }
    for (int j = 0; j < B - 1; ++j) { const u32 g = (wb + (u32)j < N) ? T[wb + j] : 255u; cache[j] = packed_cache ? (g & 3u) : g; }
#define SUB(g, q, qq) (qtab ? (((u8)(g) == (q)) ? qtab[2 * (qq)] : qtab[2 * (qq) + 1]) : (((u8)(g) == (q)) ? S->match : S->mismatch))
    for (u32 i = wb; i < we; ++i)
    {
        const u8 q = P[i];
        const u8 qq = Q ? Q[i] : 0;
        {
            F[0] = imax(F[1] + Ge, H[1] + Go);
            const u32 g = cache[0];
            i32 h = imax(F[0], H[0] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + 1, i + 1); }
            H[0] = h;
        }
        i32 E = H[0] + Go;
        for (int j = 1; j < B - 1; ++j)
        {
            F[j] = imax(F[j + 1] + Ge, H[j + 1] + Go);
            const u32 g = cache[j]; cache[j - 1] = g;
            i32 h = imax(imax(F[j], E), H[j] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + (u32)j + 1, i + 1); }
            H[j] = h;
            E = imax(h + Go, E + Ge);
        }
        const u8 g = (i + (u32)B - 1 < N) ? T[i + B - 1] : 255u;
        cache[B - 2] = packed_cache ? (g & 3u) : g;
        {
            F[B - 1] = INF;
            i32 h = imax(E, H[B - 1] + SUB(g, q, qq));
            if (type == 1) { h = imax(h, 0); sink_report(&best, &bx, &by, h, i + (u32)B, i + 1); }
            H[B - 1] = h;
        }
    }
#undef SUB
    *best_io = best; *bx_io = bx; *by_io = by;
    if (we < M)
    {
        i32 mx = H[0];
        for (int j = 1; j < B; ++j) mx = imax(mx, H[j]);
        const long long thr = (long long)min_score + (long long)(M - we) * (qtab ? qtab[0] : S->match);
        if ((long long)mx < thr) return 0;
    }
    for (int j = 0; j < B; ++j) { ckpt[2 * j] = (short)imax(H[j], SHRT_MIN + 32); ckpt[2 * j + 1] = (short)imax(F[j], SHRT_MIN + 32); }
    if (we == M)
    {
        if (type == 0) sink_report(&best, &bx, &by, H[B - 1], M + (u32)B - 1, M);
        else if (type == 2)
        {
            const u32 lim = (M + (u32)B - 1 < N ? M + (u32)B - 1 : N) - (M - 1);
            sink_report(&best, &bx, &by, H[0], M, M);
            for (int j = 1; j < B; ++j) if ((u32)j < lim) sink_report(&best, &bx, &by, H[j], M + (u32)j, M);
        }
        *best_io = best; *bx_io = bx; *by_io = by;
    }
    return 1;
}

/* window [wb, min(we, M)) of every alignment still alive; score/sink/ckpt/alive are in/out arrays (wb == 0 initialises them) */
void orc_banded_gotoh_window(int B, int type, const orc_scheme* S, const i32* qtab,
                             const u8* pat, const u8* qual, const u32* p_off, const u32* p_len,
                             const u8* txt, const u32* t_off, const u32* t_len, u32 n, u32 wb, u32 we, const i32* min_score,
                             short* ckpt, i32* score, u32* sink_x, u32* sink_y, u8* alive)
{
    for (u32 i = 0; i < n; ++i)
    {
        if (wb == 0) { score[i] = ORC_SINK_MIN; sink_x[i] = sink_y[i] = 0xFFFFFFFFu; alive[i] = 1; }
        if (!alive[i] || wb >= p_len[i]) continue;
        const u32 e = we < p_len[i] ? we : p_len[i];
        alive[i] = (u8)orc_banded_gotoh_window_one(B, type, S, qtab, pat + p_off[i], qual ? qual + p_off[i] : NULL, p_len[i],
                                                   txt + t_off[i], t_len[i], wb, e, min_score ? min_score[i] : INT_MIN,
                                                   ckpt + (size_t)i * 2 * B, &score[i], &sink_x[i], &sink_y[i]);
    }
}

/* ------------------------------------------------------------------------------------------------
 * banded Gotoh traceback (nvbio/alignment/banded_inl.h:352-489 driver; direction vectors as produced by
 * gotoh_banded_inl.h:463-620 and stored by GotohSubmatrixContext::new_cell :325-337; state machine
 * gotoh_banded_inl.h:893-958).  The reference recomputes 32-row windows between checkpoints; walking one
 * full M x B direction matrix visits the same cells with the same bits.
 * ops: the backtracer's pushes in END -> START order (0 SUBSTITUTION 'M', 1 INSERTION 'I', 2 DELETION 'D');
 * clips = (M - sink.y, source.y).  Returns the number of ops (may exceed max_ops: then truncated).
 * Substitution scores as orc_banded_gotoh_one: qtab == NULL -> the scheme's constants, else qtab[2*qq] / qtab[2*qq+1] with qq = Q[i].
 * ---------------------------------------------------------------------------------------------- */
enum { D_SUB = 0, D_INS = 1, D_DEL = 2, D_SINK = 3, D_INS_EXT = 4, D_DEL_EXT = 8 };

u32 orc_banded_traceback_one(int B, int type, const orc_scheme* S, const i32* qtab,
                             const u8* P, const u8* Q, u32 M, const u8* T, u32 N,
                             i32* out_score, u32* sink_xy, u32* source_xy, u8* ops, u32 max_ops, u32* clips)
{
    i32 best = ORC_SINK_MIN; u32 bx = 0xFFFFFFFFu, by = 0xFFFFFFFFu;
    *out_score = best; sink_xy[0] = sink_xy[1] = source_xy[0] = source_xy[1] = 0xFFFFFFFFu; clips[0] = clips[1] = 0;
    if (N < M) return 0;
    const int packed_cache = !(B == 3 || B == 5 || B == 7 || B == 15);
    const i32 Go = S->pattern_gap_open, Ge = S->pattern_gap_ext;
    const i32 INF = SHRT_MIN - imax(imax(Go, Ge), imax(S->text_gap_open, S->text_gap_ext));
    i32 H[ORC_MAX_BAND], F[ORC_MAX_BAND]; u32 cache[ORC_MAX_BAND];
    u8* dir = (u8*)malloc((size_t)(M ? M : 1) * (size_t)B);
    H[0] = 0;
    for (int j = 1; j < B; ++j) H[j] = (type == 0) ? S->text_gap_open + (j - 1) * S->text_gap_ext : 0;
    for (int j = 0; j < B; ++j) F[j] = INF;
    for (int j = 0; j < B - 1; ++j) { const u32 g = ((u32)j < N) ? T[j] : 255u; cache[j] = packed_cache ? (g & 3u) : g; }
#define SUB(g, q) (((u8)(g) == (q)) ? s_eq : s_ne)
    for (u32 i = 0; i < M; ++i)
    {
        const u8 q = P[i];
        const u8 qq = Q ? Q[i] : 0;
        const i32 s_eq = qtab ? qtab[2 * qq] : S->match, s_ne = qtab ? qtab[2 * qq + 1] : S->mismatch;
        u8 edir = D_SUB;
        {   /* j = 0 */
            const i32 ftop = F[1] + Ge, htop = H[1] + Go;
            F[0] = imax(ftop, htop);
            const u8 fdir = ftop > htop ? D_DEL_EXT : D_SUB;
            const i32 diagonal = H[0] + SUB(cache[0], q), top = F[0];
            i32 hi = imax(top, diagonal);
            u8 hdir = top > diagonal ? D_INS : D_SUB;
            if (type == 1) { hi = imax(hi, 0); if (hi == 0) hdir = D_SINK; sink_report(&best, &bx, &by, hi, i + 1, i + 1); }
            H[0] = hi;
            dir[(size_t)i * B] = (u8)(hdir | D_SUB | fdir);
        }
        i32 E = H[0] + Go;
        for (int j = 1; j < B - 1; ++j)
        {
            const i32 ftop = F[j + 1] + Ge, htop = H[j + 1] + Go;
            F[j] = imax(ftop, htop);
            const u8 fdir = ftop > htop ? D_DEL_EXT : D_SUB;
            const u32 g = cache[j]; cache[j - 1] = g;
            const i32 diagonal = H[j] + SUB(g, q), top = F[j], left = E;
            i32 hi = imax(imax(top, left), diagonal);
            u8 hdir = top > left ? (top > diagonal ? D_INS : D_SUB) : (left > diagonal ? D_DEL : D_SUB);
            if (type == 1) { hi = imax(hi, 0); if (hi == 0) hdir = D_SINK; sink_report(&best, &bx, &by, hi, i + (u32)j + 1, i + 1); }
            H[j] = hi;
            dir[(size_t)i * B + j] = (u8)(hdir | edir | fdir);
            const i32 eleft = E + Ge, ediagonal = hi + Go;
            edir = eleft > ediagonal ? D_INS_EXT : D_SUB;
            E = imax(ediagonal, eleft);
        }
        const u8 g = (i + (u32)B - 1 < N) ? T[i + B - 1] : 255u;
        cache[B - 2] = packed_cache ? (g & 3u) : g;
        {   /* j = B-1 */
            F[B - 1] = INF;
            const i32 diagonal = H[B - 1] + SUB(g, q), left = E;
            i32 hi = imax(left, diagonal);
            u8 hdir = left > diagonal ? D_DEL : D_SUB;
            if (type == 1) { hi = imax(hi, 0); if (hi == 0) hdir = D_SINK; sink_report(&best, &bx, &by, hi, i + (u32)B, i + 1); }
            H[B - 1] = hi;
            dir[(size_t)i * B + B - 1] = (u8)(hdir | edir | D_SUB);
        }
    }
#undef SUB
    if (type == 0) sink_report(&best, &bx, &by, H[B - 1], M + (u32)B - 1, M);
    else if (type == 2)
    {
        const u32 lim = (M + (u32)B - 1 < N ? M + (u32)B - 1 : N) - (M - 1);
        sink_report(&best, &bx, &by, H[0], M, M);
        for (int j = 1; j < B; ++j) if ((u32)j < lim) sink_report(&best, &bx, &by, H[j], M + (u32)j, M);
    }
    *out_score = best;
    u32 n_ops = 0;
    if (bx != 0xFFFFFFFFu && by != 0xFFFFFFFFu)
    {
        sink_xy[0] = bx; sink_xy[1] = by;
        clips[0] = M - by;
        i32 entry = (i32)(bx - by), row = (i32)by - 1;
        int state = 0;                                /* HSTATE 0, ESTATE 1, FSTATE 2 */
        int found = 0;
        u32 sx = 0, sy = 0;
        while (row >= 0)
        {
            const u8 op = dir[(size_t)row * B + entry];
            const u8 h_op = op & 3u;
            if (type == 1 && state == 0 && h_op == D_SINK) { sy = (u32)row + 1u; sx = (u32)entry + sy; found = 1; break; }
            if (state == 1)      { if ((op & D_INS_EXT) == 0) state = 0; --entry;        if (n_ops < max_ops) ops[n_ops] = D_DEL; ++n_ops; }
            else if (state == 2) { if ((op & D_DEL_EXT) == 0) state = 0; ++entry; --row; if (n_ops < max_ops) ops[n_ops] = D_INS; ++n_ops; }
            else
            {
                if (h_op == D_DEL) state = 1;
                else if (h_op == D_INS) state = 2;
                else { --row; if (n_ops < max_ops) ops[n_ops] = D_SUB; ++n_ops; }
            }
        }
        if (!found) { sy = 0; sx = (u32)entry; }
        source_xy[0] = sx; source_xy[1] = sy;
        clips[1] = sy;
    }
    free(dir);
    return n_ops;
}

void orc_banded_traceback(int B, int type, const orc_scheme* S, const i32* qtab,
                          const u8* pat, const u8* qual, const u32* p_off, const u32* p_len,
                          const u8* txt, const u32* t_off, const u32* t_len, u32 n, u32 max_ops,
                          i32* score, u32* sink_xy, u32* source_xy, u8* ops, u32* n_ops, u32* clips)
{
    for (u32 i = 0; i < n; ++i)
        n_ops[i] = orc_banded_traceback_one(B, type, S, qtab, pat + p_off[i], qual ? qual + p_off[i] : NULL, p_len[i], txt + t_off[i], t_len[i],
                                            &score[i], &sink_xy[2 * i], &source_xy[2 * i], ops + (size_t)i * max_ops, max_ops, &clips[2 * i]);
}

/* ------------------------------------------------------------------------------------------------
 * full-matrix Gotoh score (SURVEY 8f-3): aln::alignment_score with GotohAligner<TYPE,scheme,PatternBlockingTag>
 * (nvbio/alignment/gotoh/gotoh_inl.h:459-960; first column :75-89, top row :688-696, infimum :665).
 * Rows r = 1..N follow the TEXT, columns c = 1..M the PATTERN; E runs along the pattern, F along the text, both with
 * the PATTERN gap costs; the first column uses the TEXT gap costs (GLOBAL only).  sink = (text end, pattern end).
 * LOCAL reports every cell stripe by stripe (stripes of 8 pattern columns, gotoh_bandlen_selector :1491-1495), inside
 * a stripe row by row, so ties resolve to the last maximal cell in (stripe, row, column) order; SEMI_GLOBAL reports
 * H[r][M] for every row; GLOBAL reports H[N][M].  Requires M >= 1, N >= 1.
 * ---------------------------------------------------------------------------------------------- */
void orc_gotoh_full_one(int type, const orc_scheme* S, const i32* qtab, const u8* P, const u8* Q, u32 M, const u8* T, u32 N,
                        i32* out_score, u32* out_x, u32* out_y)
{
    i32 best = ORC_SINK_MIN; u32 bx = 0xFFFFFFFFu, by = 0xFFFFFFFFu;
    const i32 Go = S->pattern_gap_open, Ge = S->pattern_gap_ext;
    const i32 INF = SHRT_MIN - (Go < Ge ? Go : Ge);
    const size_t W = (size_t)M + 1;
    i32* H = (i32*)malloc(sizeof(i32) * (N + 1) * W);
    i32* E = (i32*)malloc(sizeof(i32) * (N + 1) * W);
    i32* F = (i32*)malloc(sizeof(i32) * (N + 1) * W);
    for (u32 c = 0; c <= M; ++c) { H[c] = (type != 1) ? (c > 0 ? Go + Ge * (i32)(c - 1) : 0) : 0; F[c] = INF; E[c] = INF; }
    for (u32 r = 1; r <= N; ++r)
    {
        H[r * W] = (type == 0) ? S->text_gap_open + S->text_gap_ext * (i32)(r - 1) : 0;
        E[r * W] = (type == 1) ? 0 : INF;
        F[r * W] = INF;
        for (u32 c = 1; c <= M; ++c)
        {
            const i32 f = imax(F[(r - 1) * W + c] + Ge, H[(r - 1) * W + c] + Go);
            const i32 e = imax(E[r * W + c - 1] + Ge, H[r * W + c - 1] + Go);
            const i32 s_eq = qtab ? qtab[2 * (Q ? Q[c - 1] : 0)] : S->match, s_ne = qtab ? qtab[2 * (Q ? Q[c - 1] : 0) + 1] : S->mismatch;
            const i32 d = H[(r - 1) * W + c - 1] + ((T[r - 1] == P[c - 1]) ? s_eq : s_ne);
            i32 h = imax(imax(e, f), d);
            if (type == 1) h = imax(h, 0);
            F[r * W + c] = f; E[r * W + c] = e; H[r * W + c] = h;
        }
    }
    if (type == 1)
    {
        for (u32 b = 0; b < M; b += 8)
            for (u32 r = 1; r <= N; ++r)
                for (u32 c = b + 1; c <= b + 8 && c <= M; ++c)
                    sink_report(&best, &bx, &by, H[r * W + c], r, c);
    }
    else if (type == 2) { for (u32 r = 1; r <= N; ++r) sink_report(&best, &bx, &by, H[r * W + M], r, M); }
    else sink_report(&best, &bx, &by, H[N * W + M], N, M);
    free(H); free(E); free(F);
    *out_score = best; *out_x = bx; *out_y = by;
}

void orc_gotoh_full(int type, const orc_scheme* S, const i32* qtab,
                    const u8* pat, const u8* qual, const u32* p_off, const u32* p_len,
                    const u8* txt, const u32* t_off, const u32* t_len, u32 n, i32* score, u32* sink_x, u32* sink_y)
{
    for (u32 i = 0; i < n; ++i)
        orc_gotoh_full_one(type, S, qtab, pat + p_off[i], qual ? qual + p_off[i] : NULL, p_len[i], txt + t_off[i], t_len[i], &score[i], &sink_x[i], &sink_y[i]);
}

/* ------------------------------------------------------------------------------------------------
 * full-matrix Gotoh traceback: aln::alignment_traceback<MAX_PATTERN_LEN,MAX_TEXT_LEN,CHECKPOINTS> with a Gotoh aligner
 * (generic driver nvbio/alignment/alignment_inl.h:365-488; direction vectors gotoh/gotoh_inl.h:514-555 + :426-446;
 * state machine gotoh/gotoh_inl.h:1806-1871).  The checkpointing of the reference only bounds its memory: here the whole
 * direction matrix is kept.  Per cell: hdir = top > left ? (top > diag ? DEL : SUB) : (left > diag ? INS : SUB) with
 * top = F (text gap, DELETION), left = E (pattern gap, INSERTION); LOCAL cells with H == 0 are SINKs; the E / F extension
 * bits say whether E / F were extended rather than opened.  Walk from the sink: H -> follow hdir; E -> push INSERTION, column-1,
 * stay in E while the bit is set; F likewise with DELETION, row-1.  SEMI_GLOBAL / GLOBAL finish along the first row
 * (INSERTIONs), GLOBAL along the first column (DELETIONs).  ops in END -> START order; clips = (M - sink.y, source.y).
 * Substitution scores as orc_gotoh_full_one (qtab / Q may be NULL).
 * ---------------------------------------------------------------------------------------------- */
u32 orc_gotoh_full_traceback_one(int type, const orc_scheme* S, const i32* qtab, const u8* P, const u8* Q, u32 M, const u8* T, u32 N,
                                 i32* out_score, u32* sink_xy, u32* source_xy, u8* ops, u32 max_ops, u32* clips)
{
    i32 best = ORC_SINK_MIN; u32 bx = 0xFFFFFFFFu, by = 0xFFFFFFFFu;
    *out_score = best; sink_xy[0] = sink_xy[1] = source_xy[0] = source_xy[1] = 0xFFFFFFFFu; clips[0] = clips[1] = 0;
    if (M == 0 || N == 0) return 0;
    const i32 Go = S->pattern_gap_open, Ge = S->pattern_gap_ext;
    const i32 INF = SHRT_MIN - (Go < Ge ? Go : Ge);
    const size_t W = (size_t)M + 1;
    i32* H = (i32*)malloc(sizeof(i32) * (N + 1) * W);
    i32* Fp = (i32*)malloc(sizeof(i32) * W);                 /* F of the previous row */
    u8* dir = (u8*)malloc((size_t)N * M);
    for (u32 c = 0; c <= M; ++c) { H[c] = (type != 1) ? (c > 0 ? Go + Ge * (i32)(c - 1) : 0) : 0; Fp[c] = INF; }
    for (u32 r = 1; r <= N; ++r)
    {
        H[r * W] = (type == 0) ? S->text_gap_open + S->text_gap_ext * (i32)(r - 1) : 0;
        i32 E = (type == 1) ? 0 : INF;
        for (u32 c = 1; c <= M; ++c)
        {
            const i32 ftop = Fp[c] + Ge, htop = H[(r - 1) * W + c] + Go;
            const i32 f = imax(ftop, htop);
            const u8 fdir = ftop > htop ? D_DEL_EXT : D_SUB;
            const i32 eleft = E + Ge, hleft = H[r * W + c - 1] + Go;
            E = imax(eleft, hleft);
            const u8 edir = eleft > hleft ? D_INS_EXT : D_SUB;
            const i32 s_eq = qtab ? qtab[2 * (Q ? Q[c - 1] : 0)] : S->match, s_ne = qtab ? qtab[2 * (Q ? Q[c - 1] : 0) + 1] : S->mismatch;
            const i32 diagonal = H[(r - 1) * W + c - 1] + ((T[r - 1] == P[c - 1]) ? s_eq : s_ne);
            const i32 top = f, left = E;
            i32 h = imax(imax(left, top), diagonal);
            if (type == 1) h = imax(h, 0);
            u8 hdir = top > left ? (top > diagonal ? D_DEL : D_SUB) : (left > diagonal ? D_INS : D_SUB);
            if (type == 1 && h == 0) hdir = D_SINK;
            Fp[c] = f; H[r * W + c] = h;
            dir[(size_t)(r - 1) * M + (c - 1)] = (u8)(hdir | edir | fdir);
        }
    }
    if (type == 1)
    {
        for (u32 b = 0; b < M; b += 8)
            for (u32 r = 1; r <= N; ++r)
                for (u32 c = b + 1; c <= b + 8 && c <= M; ++c)
                    sink_report(&best, &bx, &by, H[r * W + c], r, c);
    }
    else if (type == 2) { for (u32 r = 1; r <= N; ++r) sink_report(&best, &bx, &by, H[r * W + M], r, M); }
    else sink_report(&best, &bx, &by, H[N * W + M], N, M);
    *out_score = best;
    u32 n_ops = 0;
    if (bx != 0xFFFFFFFFu && by != 0xFFFFFFFFu)
    {
        sink_xy[0] = bx; sink_xy[1] = by;
        clips[0] = M - by;
        i32 row = (i32)bx, col = (i32)by - 1;          /* row 1-based over the text, col 0-based over the pattern */
        int state = 0;                                  /* HSTATE 0, ESTATE 1, FSTATE 2 */
        while (row > 0 && col >= 0)
        {
            const u8 op = dir[(size_t)(row - 1) * M + col];
            const u8 h_op = op & 3u;
            if (type == 1 && state == 0 && h_op == D_SINK) break;
            if (state == 1)      { if ((op & D_INS_EXT) == 0) state = 0; --col; if (n_ops < max_ops) ops[n_ops] = D_INS; ++n_ops; }
            else if (state == 2) { if ((op & D_DEL_EXT) == 0) state = 0; --row; if (n_ops < max_ops) ops[n_ops] = D_DEL; ++n_ops; }
            else
            {
                if (h_op == D_INS) state = 1;
                else if (h_op == D_DEL) state = 2;
                else { --row; --col; if (n_ops < max_ops) ops[n_ops] = D_SUB; ++n_ops; }
            }
        }
        u32 sx = (u32)row, sy = (u32)(col + 1);
        if (type != 1 && sx == 0) for (; sy > 0; --sy) { if (n_ops < max_ops) ops[n_ops] = D_INS; ++n_ops; }
        if (type == 0 && sy == 0) for (; sx > 0; --sx) { if (n_ops < max_ops) ops[n_ops] = D_DEL; ++n_ops; }
        source_xy[0] = sx; source_xy[1] = sy;
        clips[1] = sy;
    }
    free(H); free(Fp); free(dir);
    return n_ops;
}

void orc_gotoh_full_traceback(int type, const orc_scheme* S, const i32* qtab,
                              const u8* pat, const u8* qual, const u32* p_off, const u32* p_len,
                              const u8* txt, const u32* t_off, const u32* t_len, u32 n, u32 max_ops,
                              i32* score, u32* sink_xy, u32* source_xy, u8* ops, u32* n_ops, u32* clips)
{
    for (u32 i = 0; i < n; ++i)
        n_ops[i] = orc_gotoh_full_traceback_one(type, S, qtab, pat + p_off[i], qual ? qual + p_off[i] : NULL, p_len[i], txt + t_off[i], t_len[i],
                                                &score[i], &sink_xy[2 * i], &source_xy[2 * i], ops + (size_t)i * max_ops, max_ops, &clips[2 * i]);
}
